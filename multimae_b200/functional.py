"""torch.autograd.Function wrappers over the module-level C ABI (include/multimae_b200.h).

PyTorch supplies device memory, streams and the autograd tape; every FLOP runs in libmultimae_b200.so.  There is no
CPU/eager fallback: CPU tensors raise.

Gradient storage: parameters' gradients are accumulated by the kernels directly into a flat fp32 `GradArena` owned by
the model (zeroed once per forward), and the per-parameter views are what backward returns — or, in "owned" mode
(data-parallel trainer), what `p.grad` permanently aliases so the arena can be all-reduced in place.
"""
import ctypes
import os
import weakref

import torch

from . import _lib as L


def _require_cuda(t, what):
    if not t.is_cuda:
        raise L.MmaeError("multimae_b200.%s needs CUDA tensors: the path is sm_90a kernels only (no CPU fallback)" % what)


class Workspace:
    """One growable scratch buffer per (device, stream), reused by every Function launched on that stream (launches on
    one stream are ordered; the task decoders run on their own streams and must not share scratch)."""
    _bufs = {}

    @classmethod
    def get(cls, nbytes, device):
        stream = torch.cuda.current_stream(device).cuda_stream if device.type == "cuda" else 0
        key = (device.type, device.index, stream)
        buf = cls._bufs.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(int(nbytes * 1.1) + 4096, dtype=torch.uint8, device=device)
            cls._bufs[key] = buf
        return buf


# consecutive Blocks hand their residual add / gradient cast over to each other (block_stack); 0: block by block
BLOCK_CHAIN = os.environ.get("MMAE_BLOCK_CHAIN", "1") != "0"

_ARENAS = weakref.WeakSet()


def find_arena_for(params):
    """The live GradArena whose flat buffer holds EVERY gradient of `params` (each p.grad aliases one of its views), or
    None.  Lets a caller that was handed only `model.parameters()` - NativeScalerWithGradNormCount inside the unchanged
    train_one_epoch - reach the flat gradient buffer and the data-parallel reducer attached to it."""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return None
    for arena in list(_ARENAS):
        base, end = arena.flat.data_ptr(), arena.flat.data_ptr() + arena.flat.numel() * arena.flat.element_size()
        if all(g.device == arena.flat.device and base <= g.data_ptr() < end for g in grads):
            return arena
    return None


class GradArena:
    """Flat fp32 gradient storage for a list of (name, parameter); views are 32-byte aligned."""

    def __init__(self, named_params, device):
        self.offsets = {}
        off = 0
        for name, p in named_params:
            self.offsets[name] = (off, p.numel(), tuple(p.shape))
            off += (p.numel() + 7) // 8 * 8      # 32-byte slots: the bf16 twin of a slot stays 16-byte aligned (TMA)
        self.numel = off
        self.flat = torch.zeros(max(off, 4), dtype=torch.float32, device=device)
        self.views = {name: self.flat[o:o + n].view(shape) for name, (o, n, shape) in self.offsets.items()}
        self.owned = False     # True: p.grad aliases the views and backward returns None for parameters
        self.accumulating = False   # True between scaler(update_grad=False) calls: the next forward must not zero the arena
        self.reducer = None    # parallel.FlatGradReducer exchanging this arena between ranks (attach_data_parallel)
        _ARENAS.add(self)

    def zero_(self):
        self.flat.zero_()

    def begin_step(self):
        """Called by the model at the start of a training forward: one memset, unless a gradient accumulation over several
        forward/backward passes is in progress (NativeScalerWithGradNormCount(..., update_grad=False))."""
        if not self.accumulating:
            self.flat.zero_()

    def view(self, name):
        return self.views[name]


# ---------------------------------------------------------------------------------------------------------------------
# bf16 weight mirrors (FlatAdamW registers one): the model checks at the start of every forward that the registered
# twins are current, so a parameter change made through torch (load_state_dict, manual init) is picked up; writes that
# bypass the version counters (`.data`) call invalidate_mirrors()
# ---------------------------------------------------------------------------------------------------------------------
_MIRRORS = weakref.WeakSet()


def register_mirror(owner):
    _MIRRORS.add(owner)


def fresh_mirrors():
    for m in _MIRRORS:
        m.ensure_mirror_fresh()


def invalidate_mirrors():
    for m in _MIRRORS:
        m.invalidate_mirror()


# ---------------------------------------------------------------------------------------------------------------------
# Deterministic mode follows torch.use_deterministic_algorithms (warn_only=True counts as on): the model checks the flag
# where a step starts and the criteria, the scaler and the flat optimizers where they are called, and the library's
# switch (mmae_set_deterministic) is set only when the flag has changed.  A captured CUDA graph (train_step.TrainStep)
# replays the kernels it was captured with, so it keeps the mode of its capture.
# ---------------------------------------------------------------------------------------------------------------------
_deterministic = False          # the library's switch as last set here; it loads switched off


def sync_deterministic():
    global _deterministic
    want = torch.are_deterministic_algorithms_enabled()
    if want != _deterministic:
        L.check(L.lib().mmae_set_deterministic(int(want)), "mmae_set_deterministic")
        _deterministic = want


def _grad_ptr(arena, name):
    return arena.views[name].data_ptr()


def _ret_grads(arena, names, params):
    """What backward returns for parameter inputs."""
    out = []
    for n, p in zip(names, params):
        if p is None or not p.requires_grad:
            out.append(None)
            continue
        v = arena.views[n]
        if arena.owned or (p.grad is not None and p.grad.data_ptr() == v.data_ptr()):
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                p.grad = v
            out.append(None)
        else:
            out.append(v)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# transformer block
# ---------------------------------------------------------------------------------------------------------------------
def drop_path_prob(block):
    """Stochastic-depth rate that applies to `block` in this call: its DropPath rate in training mode, else 0."""
    dp = getattr(block, "drop_path", None)
    return float(dp.drop_prob or 0.0) if block.training and hasattr(dp, "drop_prob") else 0.0


def drop_path_scales(blocks, batch, device):
    """Per-sample factors of stochastic depth for one run of consecutive Blocks (multimae/multimae_utils.py:105-132).

    Returns one entry per block: None when the block drops nothing in this call (eval mode or rate 0), else the pair
    (s_attn, s_mlp) of fp32 [batch] tensors, s = floor(keep + u) / keep with keep = 1 - p and u ~ U[0, 1): 0 for a dropped
    sample, 1/keep for a kept one.  All draws come from ONE torch.rand on `device` (torch's CUDA generator), block by block,
    the attention branch before the MLP branch; no host synchronisation, so it can be captured in a CUDA graph and every
    replay draws anew."""
    probs = [drop_path_prob(b) for b in blocks]
    live = [i for i, p in enumerate(probs) if p > 0.0]
    out = [None] * len(probs)
    if not live:
        return out
    u = torch.rand((len(live), 2, batch), dtype=torch.float32, device=device)
    for j, i in enumerate(live):
        keep = 1.0 - probs[i]
        s = u[j].add_(keep).floor_().div_(keep)
        out[i] = (s[0], s[1])
    return out


def dropout_rates(block):
    """(attn_p, proj_p, mlp_p) that apply to `block` in this call: the rates of its Attention.attn_drop,
    Attention.proj_drop and Mlp.drop (multimae/multimae_utils.py:154,177,181) in training mode, else zeros."""
    if not block.training:
        return (0.0, 0.0, 0.0)
    return (float(block.attn.attn_drop.p), float(block.attn.proj_drop.p), float(block.mlp.drop.p))


def dropout_seeds(blocks, device):
    """Dropout seeds for one run of consecutive Blocks: one entry per block, None when the block drops nothing in this call,
    else a 0-dim int64 tensor on `device` from which the kernels derive the block's three masks (counter-based, nothing is
    stored).  All seeds come from ONE torch.randint on `device`; no host synchronisation, so it can be captured in a CUDA
    graph and every replay draws anew."""
    live = [i for i, b in enumerate(blocks) if any(p > 0.0 for p in dropout_rates(b))]
    out = [None] * len(blocks)
    if not live:
        return out
    seeds = torch.randint(0, 2 ** 63 - 1, (len(live),), dtype=torch.int64, device=device)
    for j, i in enumerate(live):
        out[i] = seeds[j]
    return out


def block_dropouts(blocks, device, fp32=False):
    """One entry per block: None when the block drops nothing in this call, else (attn_p, proj_p, mlp_p, seed) with the seed
    from dropout_seeds.  The fp32 tier has no dropout kernels: a live rate there raises."""
    if fp32 and any(any(p > 0.0 for p in dropout_rates(b)) for b in blocks):
        raise NotImplementedError("multimae_b200: dropout in training is not supported in the fp32 tier "
                                  "(fp32_output_adapters); set the adapter's drop rates to 0 or run it in eval mode")
    seeds = dropout_seeds(blocks, device)
    return [None if s is None else dropout_rates(b) + (s,) for b, s in zip(blocks, seeds)]


def _block_dropout_arg(drops, i, chained):
    """ctypes BlockDropout for block i of a stack, or None (no dropout) when neither its own sites nor (chained) the
    previous block's MLP site drop anything."""
    own = drops[i]
    prev = drops[i - 1] if chained and i > 0 else None
    if own is None and (prev is None or prev[2] == 0.0):
        return None
    d = L.BlockDropout()
    if own is not None:
        d.attn_p, d.proj_p, d.mlp_p, d.seed = own[0], own[1], own[2], own[3].data_ptr()
    if prev is not None and prev[2] > 0.0:
        d.prev_mlp_p, d.prev_seed = prev[2], prev[3].data_ptr()
    return d


BLOCK_PARAM_NAMES = ["norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight",
                     "attn.proj.bias", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight",
                     "mlp.fc2.bias"]


class BlockFunction(torch.autograd.Function):
    """n >= 1 consecutive Blocks (Block.forward, multimae/multimae_utils.py:229-232), one library call per block and
    direction.  A stack of them (the encoder, multimae/multimae.py:349; a decoder_transformer,
    multimae/output_adapters.py:271) hands off between consecutive blocks in the bf16 tier: the residual add that ends block
    i runs inside block i+1's first LayerNorm kernel, and block i+1's first LayerNorm backward emits the bf16 copy of the
    gradient and the fc2 bias gradient that block i's backward starts from.  n - 1 add passes and n - 1 cast + column-sum
    passes less than n one-block calls; same arithmetic.

    Stochastic depth: `scales` holds one drop_path_scales entry per block (None: factor 1).  Block i+1 also receives block
    i's s_mlp, the factor of the MLP branch it adds in front of its first LayerNorm (forward) and of the bf16 gradient it
    hands down (backward).

    Dropout: `drops` holds one block_dropouts entry per block (None: no dropout).  A block with one passes its rates and
    seed to the block calls, forward and backward; block i+1 also receives block i's mlp rate and seed, for the same
    reason it receives s_mlp.  Blocks without any pass NULL, the calls of a stack without dropout.

    args: x, metas (one dict per block, all of one shape; metas[0]["fp32"]: the fp32 tier of `fp32_output_adapters` - 3 x
    bf16 split GEMMs, fp32 attention / GELU - for one block), scales, drops, then the 12 BLOCK_PARAM_NAMES tensors of every
    block."""

    @staticmethod
    def forward(ctx, x, metas, scales, drops, *params):
        _require_cuda(x, "Block")
        lib = L.lib()
        n, P = len(metas), len(BLOCK_PARAM_NAMES)
        tier = "_f32" if metas[0].get("fp32") else ""
        B, N, D = x.shape
        H, hidden, eps = metas[0]["heads"], metas[0]["hidden"], metas[0]["eps"]
        x = x.contiguous().float()
        dev = x.device
        ws = Workspace.get(getattr(lib, "mmae_block%s_workspace_bytes" % tier)(B, N, D, H, hidden), dev)
        nbytes = getattr(lib, "mmae_block%s_saved_bytes" % tier)(B, N, D, H, hidden)
        # MLP branch output on its way to the next block
        y = torch.empty((B, N, D), dtype=torch.bfloat16, device=dev) if n > 1 else None
        out = torch.empty_like(x)
        xs, saveds = [], []
        x_ptr, add_ptr = x.data_ptr(), None
        for i in range(n):
            last = i == n - 1
            saved = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            x_sum = torch.empty_like(x) if add_ptr is not None else None
            prm = L.BlockParams(*[p.data_ptr() for p in params[i * P:(i + 1) * P]])
            s_attn, s_mlp, s_prev = _stack_scale_ptrs(scales, i)
            if tier:
                L.check(lib.mmae_block_f32_forward(x_ptr, out.data_ptr(), B, N, D, H, hidden, eps, s_attn, s_mlp,
                                                   ctypes.byref(prm), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                        "mmae_block_f32_forward")
            else:
                drop = _block_dropout_arg(drops, i, add_ptr is not None)
                L.check(lib.mmae_block_forward(x_ptr, add_ptr, L.ptr(x_sum), out.data_ptr() if last else None,
                                               None if last else y.data_ptr(), B, N, D, H, hidden, eps, s_attn, s_mlp,
                                               s_prev, ctypes.byref(drop) if drop is not None else None, ctypes.byref(prm),
                                               saved.data_ptr(), ws.data_ptr(), L.current_stream()), "mmae_block_forward")
            xs.append(x if x_sum is None else x_sum)
            saveds.append(saved)
            if not last:       # the next block's input: this block's x_mid (inside `saved`) + y
                x_ptr, add_ptr = lib.mmae_block_saved_x_mid(saved.data_ptr(), B, N, D, H, hidden), y.data_ptr()
        ctx.metas, ctx.params, ctx.dims, ctx.scales, ctx.drops = metas, params, (B, N, D, H, hidden), scales, drops
        ctx.save_for_backward(*xs, *saveds)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        metas, params = ctx.metas, ctx.params
        B, N, D, H, hidden = ctx.dims
        n, P = len(metas), len(BLOCK_PARAM_NAMES)
        tier = "_f32" if metas[0].get("fp32") else ""
        xs, saveds = ctx.saved_tensors[:n], ctx.saved_tensors[n:]
        dev = dout.device
        ws = Workspace.get(getattr(lib, "mmae_block%s_workspace_bytes" % tier)(B, N, D, H, hidden), dev)
        d = dout.contiguous().float()
        g_in = None                                                        # bf16(d) handed down by the block above
        g_bufs = [torch.empty((B, N, D), dtype=torch.bfloat16, device=dev) for _ in range(min(2, n - 1))]
        grads = [None] * (n * P)
        for i in reversed(range(n)):
            arena, prefix = metas[i]["arena"], metas[i]["prefix"]
            names = [prefix + k for k in BLOCK_PARAM_NAMES]
            blk = params[i * P:(i + 1) * P]
            prm = L.BlockParams(*[p.data_ptr() for p in blk])
            grd = L.BlockGrads(*[_grad_ptr(arena, k) for k in names])
            dx = torch.empty((B, N, D), dtype=torch.float32, device=dev)
            g_out, below_bias = None, None
            if i > 0:      # bf16(dx) + the fc2 bias gradient of the block below, from this block's first-LayerNorm backward
                g_out = g_bufs[i % len(g_bufs)]
                below_bias = _grad_ptr(metas[i - 1]["arena"], metas[i - 1]["prefix"] + "mlp.fc2.bias")
            s_attn, s_mlp, s_prev = _stack_scale_ptrs(ctx.scales, i)
            if tier:
                L.check(lib.mmae_block_f32_backward(xs[i].data_ptr(), d.data_ptr(), dx.data_ptr(), B, N, D, H, hidden,
                                                    s_attn, s_mlp, ctypes.byref(prm), ctypes.byref(grd),
                                                    saveds[i].data_ptr(), ws.data_ptr(), L.current_stream()),
                        "mmae_block_f32_backward")
            else:
                drop = _block_dropout_arg(ctx.drops, i, i > 0)
                L.check(lib.mmae_block_backward(xs[i].data_ptr(), d.data_ptr(), L.ptr(g_in), dx.data_ptr(), L.ptr(g_out),
                                                below_bias, B, N, D, H, hidden, s_attn, s_mlp, s_prev,
                                                ctypes.byref(drop) if drop is not None else None, ctypes.byref(prm),
                                                ctypes.byref(grd), saveds[i].data_ptr(), ws.data_ptr(),
                                                L.current_stream()), "mmae_block_backward")
            if metas[i].get("on_grads_ready") is not None:
                metas[i]["on_grads_ready"](names)       # fc2.bias of block i is complete: its column sums came from block i+1
            grads[i * P:(i + 1) * P] = _ret_grads(arena, names, blk)
            d, g_in = dx, g_out
        return (d, None, None, None) + tuple(grads)


def _stack_scale_ptrs(scales, i):
    """(s_attn, s_mlp, s_prev) device pointers of block i of a stack (None = factor 1); s_prev is block i-1's s_mlp."""
    own = scales[i]
    prev = scales[i - 1] if i > 0 else None
    return (None if own is None else own[0].data_ptr(), None if own is None else own[1].data_ptr(),
            None if prev is None else prev[1].data_ptr())


def block_stack(blocks, x, fp32=False):
    """Run an nn.Sequential of multimae_utils.Block as one BlockFunction with hand-offs when it applies (CUDA path, >= 2
    blocks of one shape bound to an arena, BLOCK_CHAIN on), else block by block (`fp32`: in the fp32 tier, always block by
    block).  The stochastic-depth factors and the dropout seeds of all blocks are drawn once, up front (drop_path_scales,
    block_dropouts)."""
    blocks = list(blocks)
    scales = drop_path_scales(blocks, x.shape[0], x.device)
    drops = block_dropouts(blocks, x.device, fp32)
    metas = [getattr(b, "_meta", None) for b in blocks]
    ok = (BLOCK_CHAIN and not fp32 and len(blocks) >= 2
          and all(m is not None and m["arena"].flat.device == x.device for m in metas)
          and not any(getattr(b, "_own_arena", False) for b in blocks)
          and len({(b.dim, b.num_heads, b.hidden, b.norm1.eps) for b in blocks}) == 1)
    if not ok:
        for b, sc, dr in zip(blocks, scales, drops):
            x = b.run(x, fp32=fp32, scales=sc, drops=dr)
        return x
    flat = []
    for b in blocks:
        flat += list(b._params())
    return BlockFunction.apply(x, metas, scales, drops, *flat)


# ---------------------------------------------------------------------------------------------------------------------
# gather-first patch embedding
# ---------------------------------------------------------------------------------------------------------------------
class EmbedFunction(torch.autograd.Function):
    """input adapters + token selection + global-token append (multimae/multimae.py:312-347) as one GEMM + 2 kernels.

    args: meta (dict), ids_keep, then per task [data, weight, bias, class_emb-or-None], then global_tokens, then - only when
    some position table is trainable - one pos_emb parameter (or None: frozen, its rows come in meta["pos"]) per task.
    A trainable table is resized on the device in forward (mmae_pos_resample_forward, reading the parameter in place); in
    backward its rows' gradient (mmae_embed_pos_backward, through meta["ids_restore"]) goes through the adjoint resize into
    the table's arena slot (mmae_pos_resample_backward).  meta then also carries pos_names and pos_modes, one per task."""

    @staticmethod
    def forward(ctx, meta, ids_keep, *tensors):
        lib = L.lib()
        layout = meta["layout"]
        T_tasks = layout.num_tasks
        per_task = [tensors[4 * t:4 * t + 4] for t in range(T_tasks)]
        global_tokens = tensors[4 * T_tasks]
        tables = tensors[4 * T_tasks + 1:] or (None,) * T_tasks
        B, T = ids_keep.shape
        G, D = global_tokens.shape[-2], global_tokens.shape[-1]
        _require_cuda(ids_keep, "embed")
        ins, prm = L.EmbedInputs(), L.EmbedParams()
        keep_alive = []
        pos = list(meta["pos"])
        for t, table in enumerate(tables):
            if table is not None:          # trainable: this call's rows, resized from the parameter as it is now
                _require_cuda(table, "embed")
                nh, nw = layout.grid_h[t], layout.grid_w[t]
                pos[t] = torch.empty((nh * nw, D), dtype=torch.float32, device=ids_keep.device)
                L.check(lib.mmae_pos_resample_forward(table.data_ptr(), D, table.shape[2], table.shape[3], nh, nw,
                                                      meta["pos_modes"][t], pos[t].data_ptr(), L.current_stream()),
                        "mmae_pos_resample_forward")
        for t, (data, w, b, cemb) in enumerate(per_task):
            _require_cuda(data, "embed")
            data = data.contiguous()
            if layout.is_semseg[t]:
                assert data.dtype == torch.int64
            else:
                data = data.float()
            keep_alive.append(data)
            ins.data[t] = data.data_ptr()
            ins.class_emb[t] = cemb.data_ptr() if cemb is not None else None
            prm.weight[t] = w.data_ptr()
            prm.bias[t] = b.data_ptr()
            prm.pos[t] = pos[t].data_ptr()
        prm.global_tokens = global_tokens.data_ptr()
        dev = ids_keep.device
        saved = torch.empty(lib.mmae_embed_saved_bytes(ctypes.byref(layout), B, T, D), dtype=torch.uint8, device=dev)
        ws = Workspace.get(lib.mmae_embed_workspace_bytes(ctypes.byref(layout), B, T, D), dev)
        out = torch.empty((B, T + G, D), dtype=torch.float32, device=dev)
        ids_keep = ids_keep.contiguous()
        L.check(lib.mmae_embed_forward(ctypes.byref(layout), ctypes.byref(ins), ctypes.byref(prm), ids_keep.data_ptr(), B,
                                       T, G, D, out.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_embed_forward")
        ctx.meta = meta
        ctx.tensors = tensors
        ctx.keep_alive = keep_alive
        ctx.pos = pos
        ctx.dims = (B, T, G, D)
        ctx.save_for_backward(ids_keep, saved)
        return out

    @staticmethod
    def backward(ctx, dx):
        lib = L.lib()
        ids_keep, saved = ctx.saved_tensors
        meta, tensors = ctx.meta, ctx.tensors
        layout, arena, names = meta["layout"], meta["arena"], meta["names"]
        T_tasks = layout.num_tasks
        B, T, G, D = ctx.dims
        ins, prm, grd = L.EmbedInputs(), L.EmbedParams(), L.EmbedGrads()
        flat_names, flat_params = [], []
        for t in range(T_tasks):
            data, w, b, cemb = tensors[4 * t:4 * t + 4]
            ins.data[t] = ctx.keep_alive[t].data_ptr()
            ins.class_emb[t] = cemb.data_ptr() if cemb is not None else None
            prm.weight[t] = w.data_ptr()
            prm.bias[t] = b.data_ptr()
            prm.pos[t] = ctx.pos[t].data_ptr()
            wn, bn, cn = names[t]
            grd.weight[t] = _grad_ptr(arena, wn)
            grd.bias[t] = _grad_ptr(arena, bn)
            grd.class_emb[t] = _grad_ptr(arena, cn) if cn is not None else None
            flat_names += [None, wn, bn, cn]
            flat_params += [None, w, b, cemb]
        gt = tensors[4 * T_tasks]
        prm.global_tokens = gt.data_ptr()
        grd.global_tokens = _grad_ptr(arena, "global_tokens")
        flat_names.append("global_tokens")
        flat_params.append(gt)
        ws = Workspace.get(lib.mmae_embed_workspace_bytes(ctypes.byref(layout), B, T, D), dx.device)
        dx = dx.contiguous().float()
        L.check(lib.mmae_embed_backward(ctypes.byref(layout), ctypes.byref(ins), ctypes.byref(prm), ctypes.byref(grd),
                                        ids_keep.data_ptr(), B, T, G, D, dx.data_ptr(), saved.data_ptr(), ws.data_ptr(),
                                        L.current_stream()), "mmae_embed_backward")
        tables = tensors[4 * T_tasks + 1:]
        if tables:
            _pos_backward(meta, tables, ctx.pos, dx, B, T, G, D)
            flat_names += meta["pos_names"]
            flat_params += list(tables)
        real = [(n, p) for n, p in zip(flat_names, flat_params) if n is not None]
        if meta.get("on_grads_ready") is not None:
            meta["on_grads_ready"]([n for n, _ in real])
        rets = iter(_ret_grads(arena, [n for n, _ in real], [p for _, p in real]))
        out = [None if n is None else next(rets) for n in flat_names]
        return (None, None) + tuple(out)


def _pos_backward(meta, tables, rows, dx, B, T, G, D):
    """Gradient of the trainable position tables of one EmbedFunction call, accumulated into their arena slots: the rows'
    gradient of every trainable task in one pass over dx, then one adjoint resize per table."""
    lib = L.lib()
    layout, arena, ids_restore = meta["layout"], meta["arena"], meta["ids_restore"]
    drows = [None if tb is None else torch.empty_like(r) for tb, r in zip(tables, rows)]
    arr = (ctypes.c_void_p * layout.num_tasks)(*[L.ptr(g) for g in drows])
    L.check(lib.mmae_embed_pos_backward(ctypes.byref(layout), ids_restore.data_ptr(), B, T, G, D, dx.data_ptr(), arr,
                                        L.current_stream()), "mmae_embed_pos_backward")
    for t, (tb, g) in enumerate(zip(tables, drows)):
        if tb is not None:
            L.check(lib.mmae_pos_resample_backward(g.data_ptr(), D, tb.shape[2], tb.shape[3], layout.grid_h[t],
                                                   layout.grid_w[t], meta["pos_modes"][t],
                                                   _grad_ptr(arena, meta["pos_names"][t]), L.current_stream()),
                    "mmae_pos_resample_backward")


# ---------------------------------------------------------------------------------------------------------------------
# decoder head / tail
# ---------------------------------------------------------------------------------------------------------------------
HEAD_PARAM_NAMES = ["proj_context.weight", "proj_context.bias", "mask_token", "context_norm.weight", "context_norm.bias",
                    "query_norm.weight", "query_norm.bias", "out_norm.weight", "out_norm.bias", "decoder.q.weight",
                    "decoder.q.bias", "decoder.kv.weight", "decoder.kv.bias", "decoder.proj.weight",
                    "decoder.proj.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias"]


class SharedContextFunction(torch.autograd.Function):
    """proj_context (multimae/output_adapters.py:258) of every half-precision output adapter as ONE GEMM on the encoder
    output they all receive (multimae/multimae.py:357-366): enc [B, Nc, De] -> ctx [B*Nc, sum_i Dd_i] fp32; adapter i reads
    its column segment through DecoderHeadFunction (meta["shared"]).

    args: enc, meta, then (proj_context.weight, proj_context.bias) per adapter.  meta: arena, weight_names (arena names of
    the weights), on_grads_ready, state (dict shared with the heads).  Backward protocol: each head writes its bf16 context
    gradient into its segment of state["dctx"] and appends a completion event to state["events"] (the heads run on their
    own streams); it returns no gradient for `ctx`, so autograd calls this backward - after all heads - with None, and the
    weight-gradient GEMM and the ONE input-gradient GEMM run here.  The bias gradients are produced by the heads."""

    @staticmethod
    def forward(ctx, enc, meta, *wb):
        _require_cuda(enc, "proj_context")
        ctx.set_materialize_grads(False)
        lib = L.lib()
        enc = enc.contiguous().float()
        B, Nc, De = enc.shape
        rows = B * Nc
        weights = wb[0::2]
        prm = L.CtxProjParams()
        prm.num = len(weights)
        for i, (w, b) in enumerate(zip(weights, wb[1::2])):
            prm.dim[i], prm.weight[i], prm.bias[i] = w.shape[0], w.data_ptr(), b.data_ptr()
        dsum = sum(w.shape[0] for w in weights)
        saved = torch.empty(lib.mmae_ctxproj_saved_bytes(rows, De, dsum), dtype=torch.uint8, device=enc.device)
        out = torch.empty((rows, dsum), dtype=torch.float32, device=enc.device)
        L.check(lib.mmae_ctxproj_forward(enc.data_ptr(), rows, De, ctypes.byref(prm), out.data_ptr(), saved.data_ptr(),
                                         L.current_stream()), "mmae_ctxproj_forward")
        state = meta["state"]
        state["events"] = []
        # zero-filled: the segment of an adapter whose prediction does not reach the loss is never written
        state["dctx"] = (torch.zeros((rows, dsum), dtype=torch.bfloat16, device=enc.device)
                         if any(ctx.needs_input_grad) else None)
        ctx.meta, ctx.wb, ctx.dims = meta, wb, (B, Nc, De, dsum)
        ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, _unused):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta, wb = ctx.meta, ctx.wb
        B, Nc, De, dsum = ctx.dims
        state, arena, names = meta["state"], meta["arena"], meta["weight_names"]
        weights = wb[0::2]
        if saved.is_cuda:                          # the heads ran their backward on the task decoders' streams
            cur = torch.cuda.current_stream()
            for ev in state["events"]:
                cur.wait_event(ev)
        state["events"] = []
        prm, grd = L.CtxProjParams(), L.CtxProjGrads()
        prm.num = len(weights)
        for i, (w, b) in enumerate(zip(weights, wb[1::2])):
            prm.dim[i], prm.weight[i], prm.bias[i] = w.shape[0], w.data_ptr(), b.data_ptr()
            grd.weight[i] = _grad_ptr(arena, names[i])
        denc = torch.empty((B, Nc, De), dtype=torch.float32, device=saved.device)
        L.check(lib.mmae_ctxproj_backward(B * Nc, De, ctypes.byref(prm), ctypes.byref(grd), state["dctx"].data_ptr(),
                                          denc.data_ptr(), saved.data_ptr(), L.current_stream()), "mmae_ctxproj_backward")
        state["dctx"] = None
        if meta.get("on_grads_ready") is not None:
            meta["on_grads_ready"](list(names))
        gw = _ret_grads(arena, names, weights)
        out = []
        for g in gw:
            out += [g, None]                       # bias gradients: DecoderHeadFunction
        return (denc, None) + tuple(out)


def _fill_head_struct(st, vals, task_vals):
    """vals follow HEAD_PARAM_NAMES order; task_vals is the per-context-task pointer list."""
    (st.proj_context_w, st.proj_context_b, st.mask_token, st.context_norm_w, st.context_norm_b, st.query_norm_w,
     st.query_norm_b, st.out_norm_w, st.out_norm_b, st.q_w, st.q_b, st.kv_w, st.kv_b, st.proj_w, st.proj_b, st.fc1_w,
     st.fc1_b, st.fc2_w, st.fc2_b) = vals
    for t, v in enumerate(task_vals):
        st.task_emb[t] = v


class DecoderHeadFunction(torch.autograd.Function):
    """proj_context .. x + mlp(out_norm(x)) of SpatialOutputAdapter.forward (multimae/output_adapters.py:258-266).

    args: enc, meta, ids_keep, ids_restore, then the 19 HEAD_PARAM_NAMES tensors, then one task embedding (or None)
    per context task.  With meta["shared"] (dict: offset, ld, state, enc_shape) `enc` is the output of
    SharedContextFunction instead, proj_context.weight is passed as None, and the head starts / ends at its column
    segment of the shared projection / gradient matrix."""

    @staticmethod
    def forward(ctx, enc, meta, ids_keep, ids_restore, *params):
        _require_cuda(enc, "SpatialOutputAdapter")
        lib = L.lib()
        shared = meta.get("shared")
        if shared is None:
            enc = enc.contiguous().float()
            B, Nc, De = enc.shape
        else:
            assert not meta.get("fp32") and enc.dtype == torch.float32 and enc.is_contiguous()
            B, Nc, De = shared["enc_shape"]
        ix = L.DecoderIndex()
        ix.batch, ix.dim, ix.num_global = B, meta["dim"], meta["num_global"]
        ix.num_visible = Nc - meta["num_global"]
        ix.num_queries, ix.total_tokens = meta["num_queries"], meta["tok_offset"][-1]
        ix.num_tasks, ix.own_task = len(meta["tok_offset"]) - 1, meta["own_task"]
        ix.query_mode = meta.get("query_mode", 0)
        for i, o in enumerate(meta["tok_offset"]):
            ix.tok_offset[i] = o
        ids_keep = ids_keep.contiguous()
        ids_restore = ids_restore.contiguous()
        ix.ids_keep, ix.ids_restore = ids_keep.data_ptr(), ids_restore.data_ptr()
        H, hidden, eps = meta["heads"], meta["hidden"], meta["eps"]
        main, task = params[:len(HEAD_PARAM_NAMES)], params[len(HEAD_PARAM_NAMES):]
        prm = L.DecHeadParams()
        _fill_head_struct(prm, [L.ptr(p) for p in main], [None if p is None else p.data_ptr() for p in task])
        prm.pos = meta["pos"].data_ptr()
        f32 = "_f32" if meta.get("fp32") else ""
        De_q = De if shared is None else 0            # *_ctx heads hold no encoder copy / proj_context operand
        saved = torch.empty(getattr(lib, "mmae_dechead%s_saved_bytes" % f32)(ctypes.byref(ix), De_q, H, hidden),
                            dtype=torch.uint8, device=enc.device)
        ws = Workspace.get(getattr(lib, "mmae_dechead%s_workspace_bytes" % f32)(ctypes.byref(ix), De_q, H, hidden), enc.device)
        out = torch.empty((B, ix.num_queries, ix.dim), dtype=torch.float32, device=enc.device)
        if shared is None:
            L.check(getattr(lib, "mmae_dechead%s_forward" % f32)(enc.data_ptr(), De, ctypes.byref(ix), H, hidden, eps,
                                                                 ctypes.byref(prm), out.data_ptr(), saved.data_ptr(),
                                                                 ws.data_ptr(), L.current_stream()),
                    "mmae_dechead%s_forward" % f32)
        else:
            L.check(lib.mmae_dechead_forward_ctx(enc.data_ptr() + 4 * shared["offset"], shared["ld"], ctypes.byref(ix), H,
                                                 hidden, eps, ctypes.byref(prm), out.data_ptr(), saved.data_ptr(),
                                                 ws.data_ptr(), L.current_stream()), "mmae_dechead_forward_ctx")
        ctx.meta, ctx.params, ctx.ix, ctx.enc_shape = meta, params, ix, (B, Nc, De)
        # the shared projection is not needed again: queries / context are in `saved`
        ctx.save_for_backward(enc if shared is None else enc.new_empty(0), saved, ids_keep, ids_restore)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        enc, saved, ids_keep, ids_restore = ctx.saved_tensors
        meta, params, ix = ctx.meta, ctx.params, ctx.ix
        B, Nc, De = ctx.enc_shape
        shared = meta.get("shared")
        H, hidden = meta["heads"], meta["hidden"]
        arena, prefix = meta["arena"], meta["prefix"]
        main, task = params[:len(HEAD_PARAM_NAMES)], params[len(HEAD_PARAM_NAMES):]
        names = [prefix + n for n in HEAD_PARAM_NAMES]
        task_names = [None if p is None else prefix + "task_embeddings." + tn for p, tn in zip(task, meta["task_names"])]
        prm, grd = L.DecHeadParams(), L.DecHeadGrads()
        _fill_head_struct(prm, [L.ptr(p) for p in main], [None if p is None else p.data_ptr() for p in task])
        prm.pos = meta["pos"].data_ptr()
        # main[0] (proj_context.weight) is None under the shared projection: its gradient belongs to SharedContextFunction
        _fill_head_struct(grd, [None if p is None else _grad_ptr(arena, n) for n, p in zip(names, main)],
                          [None if n is None else _grad_ptr(arena, n) for n in task_names])
        f32 = "_f32" if meta.get("fp32") else ""
        De_q = De if shared is None else 0
        ws = Workspace.get(getattr(lib, "mmae_dechead%s_workspace_bytes" % f32)(ctypes.byref(ix), De_q, H, hidden), dout.device)
        dout = dout.contiguous().float()
        if shared is None:
            denc = torch.zeros_like(enc)
            L.check(getattr(lib, "mmae_dechead%s_backward" % f32)(enc.data_ptr(), De, ctypes.byref(ix), H, hidden,
                                                                  ctypes.byref(prm), ctypes.byref(grd), dout.data_ptr(),
                                                                  denc.data_ptr(), saved.data_ptr(), ws.data_ptr(),
                                                                  L.current_stream()), "mmae_dechead%s_backward" % f32)
        else:
            denc, state = None, shared["state"]
            L.check(lib.mmae_dechead_backward_ctx(ctypes.byref(ix), H, hidden, ctypes.byref(prm), ctypes.byref(grd),
                                                  dout.data_ptr(), state["dctx"].data_ptr() + 2 * shared["offset"],
                                                  shared["ld"], saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                    "mmae_dechead_backward_ctx")
            if dout.is_cuda:
                state["events"].append(torch.cuda.current_stream().record_event())
            names = [n for n, p in zip(names, main) if p is not None]
            main = tuple(p for p in main if p is not None)
        all_names = names + [n for n in task_names if n is not None]
        if meta.get("on_grads_ready") is not None:
            meta["on_grads_ready"](all_names)
        g_main = _ret_grads(arena, names, main)
        if shared is not None:
            g_main = [None] + list(g_main)             # the slot of proj_context.weight (passed as None)
        g_task = [None if n is None else _ret_grads(arena, [n], [p])[0] for n, p in zip(task_names, task)]
        return (denc, None, None, None) + tuple(g_main) + tuple(g_task)


class DecoderTailFunction(torch.autograd.Function):
    """out_proj + un-patchify (multimae/output_adapters.py:274-280)."""

    @staticmethod
    def forward(ctx, x, meta, weight, bias):
        _require_cuda(x, "SpatialOutputAdapter")
        lib = L.lib()
        x = x.contiguous().float()
        B, _, Dd = x.shape
        nh, nw, C, P = meta["nh"], meta["nw"], meta["channels"], meta["patch"]
        pred = torch.empty((B, C, nh * P, nw * P), dtype=torch.float32, device=x.device)
        if meta.get("fp32"):      # fp32 tier: the input itself is what backward needs
            ws = Workspace.get(lib.mmae_dectail_f32_workspace_bytes(B, nh, nw, Dd, C, P), x.device)
            L.check(lib.mmae_dectail_f32_forward(x.data_ptr(), B, nh, nw, Dd, C, P, weight.data_ptr(), bias.data_ptr(),
                                                 pred.data_ptr(), ws.data_ptr(), L.current_stream()), "mmae_dectail_f32_forward")
            saved = x
        else:
            saved = torch.empty(lib.mmae_dectail_saved_bytes(B, nh, nw, Dd, C, P), dtype=torch.uint8, device=x.device)
            ws = Workspace.get(lib.mmae_dectail_workspace_bytes(B, nh, nw, Dd, C, P), x.device)
            L.check(lib.mmae_dectail_forward(x.data_ptr(), B, nh, nw, Dd, C, P, weight.data_ptr(), bias.data_ptr(),
                                             pred.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                    "mmae_dectail_forward")
        ctx.meta, ctx.dims, ctx.params = meta, (B, nh, nw, Dd, C, P), (weight, bias)
        ctx.save_for_backward(saved)
        return pred

    @staticmethod
    def backward(ctx, dpred):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta = ctx.meta
        B, nh, nw, Dd, C, P = ctx.dims
        weight, bias = ctx.params
        arena, prefix = meta["arena"], meta["prefix"]
        names = [prefix + "out_proj.weight", prefix + "out_proj.bias"]
        dpred = dpred.contiguous().float()
        dx = torch.empty((B, nh * nw, Dd), dtype=torch.float32, device=dpred.device)
        if meta.get("fp32"):
            ws = Workspace.get(lib.mmae_dectail_f32_workspace_bytes(B, nh, nw, Dd, C, P), dpred.device)
            L.check(lib.mmae_dectail_f32_backward(saved.data_ptr(), dpred.data_ptr(), B, nh, nw, Dd, C, P, weight.data_ptr(),
                                                  _grad_ptr(arena, names[0]), _grad_ptr(arena, names[1]), dx.data_ptr(),
                                                  ws.data_ptr(), L.current_stream()), "mmae_dectail_f32_backward")
        else:
            ws = Workspace.get(lib.mmae_dectail_workspace_bytes(B, nh, nw, Dd, C, P), dpred.device)
            L.check(lib.mmae_dectail_backward(dpred.data_ptr(), B, nh, nw, Dd, C, P, weight.data_ptr(),
                                              _grad_ptr(arena, names[0]), _grad_ptr(arena, names[1]), dx.data_ptr(),
                                              saved.data_ptr(), ws.data_ptr(), L.current_stream()), "mmae_dectail_backward")
        if meta.get("on_grads_ready") is not None:
            meta["on_grads_ready"](names)
        gw, gb = _ret_grads(arena, names, [weight, bias])
        return dx, None, gw, gb


# ---------------------------------------------------------------------------------------------------------------------
# classification head
# ---------------------------------------------------------------------------------------------------------------------
CLS_PARAM_NAMES = ["norm.weight", "norm.bias", "head.weight", "head.bias"]


class ClsHeadFunction(torch.autograd.Function):
    """LinearOutputAdapter.forward (multimae/output_adapters.py:345-356): token pool -> LayerNorm -> Linear as one call each
    way (mmae_clshead_forward / _backward).

    args: x [B, N, D], meta, norm.weight, norm.bias, head.weight, head.bias (both None when num_classes = 0).  meta: arena,
    prefix, on_grads_ready, num_classes, mean_pool, eps, save (False: no backward will follow - the saved tensors live in
    the stream's scratch buffer instead of a fresh allocation)."""

    @staticmethod
    def forward(ctx, x, meta, norm_w, norm_b, head_w, head_b):
        _require_cuda(x, "LinearOutputAdapter")
        lib = L.lib()
        x = x.contiguous().float()
        B, N, D = x.shape
        C, mean_pool = meta["num_classes"], int(bool(meta["mean_pool"]))
        out = torch.empty((B, C if C > 0 else D), dtype=torch.float32, device=x.device)
        nsaved = lib.mmae_clshead_saved_bytes(B, N, D, C)
        nws = lib.mmae_clshead_workspace_bytes(B, N, D, C)
        if meta["save"]:
            saved = torch.empty(nsaved, dtype=torch.uint8, device=x.device)
            ws = Workspace.get(nws, x.device)
            saved_ptr, ws_ptr = saved.data_ptr(), ws.data_ptr()
        else:
            ws = Workspace.get(nws + 256 + nsaved, x.device)
            ws_ptr = ws.data_ptr()
            saved, saved_ptr = None, (ws_ptr + nws + 255) // 256 * 256
        L.check(lib.mmae_clshead_forward(x.data_ptr(), B, N, D, C, mean_pool, float(meta["eps"]), norm_w.data_ptr(),
                                         norm_b.data_ptr(), L.ptr(head_w), L.ptr(head_b), out.data_ptr(), saved_ptr,
                                         ws_ptr, L.current_stream()), "mmae_clshead_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, (B, N, D, C, mean_pool), (norm_w, norm_b, head_w, head_b)
            ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta, params = ctx.meta, ctx.params
        B, N, D, C, mean_pool = ctx.dims
        arena, prefix = meta["arena"], meta["prefix"]
        names = [prefix + n for n in CLS_PARAM_NAMES]
        grd = [None if p is None else _grad_ptr(arena, n) for n, p in zip(names, params)]
        ws = Workspace.get(lib.mmae_clshead_workspace_bytes(B, N, D, C), dout.device)
        dout = dout.contiguous().float()
        dx = torch.empty((B, N, D), dtype=torch.float32, device=dout.device)
        L.check(lib.mmae_clshead_backward(dout.data_ptr(), B, N, D, C, mean_pool, params[0].data_ptr(), L.ptr(params[2]),
                                          *grd, dx.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_clshead_backward")
        if meta.get("on_grads_ready") is not None:
            meta["on_grads_ready"]([n for n, p in zip(names, params) if p is not None])
        return (dx, None) + tuple(_ret_grads(arena, names, params))


# ---------------------------------------------------------------------------------------------------------------------
# semantic-segmentation head (ConvNeXtAdapter): proj -> block x depth -> tail, each one call each way
# ---------------------------------------------------------------------------------------------------------------------
CONVNEXT_BLOCK_PARAM_NAMES = ["dwconv.weight", "dwconv.bias", "norm.weight", "norm.bias", "pwconv1.weight", "pwconv1.bias",
                              "pwconv2.weight", "pwconv2.bias"]


def _saved_and_ws(meta, nsaved, nws, device):
    """`saved` as a fresh tensor kept for backward, or - under torch.no_grad() (meta["save"] False) - carved from the stream's
    scratch buffer behind the workspace, so that nothing outlives the call."""
    if meta["save"]:
        saved = torch.empty(nsaved, dtype=torch.uint8, device=device)
        return saved, saved.data_ptr(), Workspace.get(nws, device).data_ptr()
    ws_ptr = Workspace.get(nws + 256 + nsaved, device).data_ptr()
    return None, (ws_ptr + nws + 255) // 256 * 256, ws_ptr


def _report(meta, names, params):
    if meta.get("on_grads_ready") is not None:
        meta["on_grads_ready"]([n for n, p in zip(names, params) if p is not None])
    return _ret_grads(meta["arena"], names, params)


class ConvNeXtProjFunction(torch.autograd.Function):
    """Token gather + proj_dec of ConvNeXtAdapter.forward (multimae/output_adapters.py:545-562): encoder tokens [B, N, D] ->
    the fp32 feature map as its [B*n*s*s, C] channels-last view (mmae_convnext_proj_*).

    args: enc, meta, proj_dec.weight, proj_dec.bias.  meta: arena, prefix, on_grads_ready, save, n (tokens per task),
    starts (first token of each main task), channels (C)."""

    @staticmethod
    def forward(ctx, enc, meta, weight, bias):
        _require_cuda(enc, "ConvNeXtAdapter")
        lib = L.lib()
        enc = enc.contiguous().float()
        B, N, D = enc.shape
        n, starts, E = meta["n"], list(meta["starts"]), weight.shape[0]
        arr = (ctypes.c_int * len(starts))(*starts)
        saved, saved_ptr, ws_ptr = _saved_and_ws(meta, lib.mmae_convnext_proj_saved_bytes(B, n, D * len(starts), E),
                                                 lib.mmae_convnext_proj_workspace_bytes(B, n, D * len(starts), E), enc.device)
        out = torch.empty((B * n * E // meta["channels"], meta["channels"]), dtype=torch.float32, device=enc.device)
        L.check(lib.mmae_convnext_proj_forward(enc.data_ptr(), B, N, D, n, len(starts), arr, E, weight.data_ptr(),
                                               bias.data_ptr(), out.data_ptr(), saved_ptr, ws_ptr, L.current_stream()),
                "mmae_convnext_proj_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, (B, N, D), (weight, bias)
            ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta, (weight, bias) = ctx.meta, ctx.params
        B, N, D = ctx.dims
        n, starts, E = meta["n"], list(meta["starts"]), weight.shape[0]
        arr = (ctypes.c_int * len(starts))(*starts)
        names = [meta["prefix"] + "proj_dec.weight", meta["prefix"] + "proj_dec.bias"]
        ws = Workspace.get(lib.mmae_convnext_proj_workspace_bytes(B, n, D * len(starts), E), dout.device)
        dout = dout.contiguous().float()
        denc = torch.empty((B, N, D), dtype=torch.float32, device=dout.device)
        L.check(lib.mmae_convnext_proj_backward(dout.data_ptr(), B, N, D, n, len(starts), arr, E, weight.data_ptr(),
                                                _grad_ptr(meta["arena"], names[0]), _grad_ptr(meta["arena"], names[1]),
                                                denc.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_convnext_proj_backward")
        return (denc, None) + tuple(_report(meta, names, [weight, bias]))


class ConvNeXtBlockFunction(torch.autograd.Function):
    """ConvNeXtBlock.forward (multimae/output_adapter_utils.py:47-57, gamma None, drop_path 0) on the [P, C] view
    (mmae_convnext_block_*).  args: x, meta (as ConvNeXtProjFunction plus nh, nw, s, eps; prefix ends in "blocks.<i>."),
    then the 8 CONVNEXT_BLOCK_PARAM_NAMES tensors - the order of the entry points' pointer arrays."""

    @staticmethod
    def forward(ctx, x, meta, *params):
        _require_cuda(x, "ConvNeXtAdapter")
        lib = L.lib()
        x = x.contiguous().float()
        dims = (meta["B"], meta["nh"], meta["nw"], meta["s"], x.shape[1])
        saved, saved_ptr, ws_ptr = _saved_and_ws(meta, lib.mmae_convnext_block_saved_bytes(*dims),
                                                 lib.mmae_convnext_block_workspace_bytes(*dims), x.device)
        out = torch.empty_like(x)
        prm = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        L.check(lib.mmae_convnext_block_forward(x.data_ptr(), out.data_ptr(), *dims, float(meta["eps"]), prm,
                                                saved_ptr, ws_ptr, L.current_stream()), "mmae_convnext_block_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, dims, params
            ctx.save_for_backward(x, saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        x, saved = ctx.saved_tensors
        meta, dims, params = ctx.meta, ctx.dims, ctx.params
        names = [meta["prefix"] + n for n in CONVNEXT_BLOCK_PARAM_NAMES]
        ws = Workspace.get(lib.mmae_convnext_block_workspace_bytes(*dims), dout.device)
        dout = dout.contiguous().float()
        dx = torch.empty_like(x)
        prm = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        grd = (ctypes.c_void_p * len(names))(*[_grad_ptr(meta["arena"], n) for n in names])
        L.check(lib.mmae_convnext_block_backward(x.data_ptr(), dout.data_ptr(), dx.data_ptr(), *dims, prm, grd,
                                                 saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_convnext_block_backward")
        return (dx, None) + tuple(_report(meta, names, params))


class ConvNeXtTailFunction(torch.autograd.Function):
    """final_layer + bilinear upsample of ConvNeXtAdapter.forward (multimae/output_adapters.py:570-573): [P, C] ->
    [B, K, H, W] fp32 (mmae_convnext_tail_*).  args: x, meta (plus num_classes, H, W), final_layer.weight, .bias."""

    @staticmethod
    def forward(ctx, x, meta, weight, bias):
        _require_cuda(x, "ConvNeXtAdapter")
        lib = L.lib()
        x = x.contiguous().float()
        K, H, W = meta["num_classes"], meta["H"], meta["W"]
        dims = (meta["B"], meta["nh"], meta["nw"], meta["s"], x.shape[1], K)
        saved, saved_ptr, ws_ptr = _saved_and_ws(meta, lib.mmae_convnext_tail_saved_bytes(*dims),
                                                 lib.mmae_convnext_tail_workspace_bytes(*dims), x.device)
        out = torch.empty((meta["B"], K, H, W), dtype=torch.float32, device=x.device)
        L.check(lib.mmae_convnext_tail_forward(x.data_ptr(), *dims, H, W, weight.data_ptr(), bias.data_ptr(), out.data_ptr(),
                                               saved_ptr, ws_ptr, L.current_stream()), "mmae_convnext_tail_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, dims, (weight, bias)
            ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta, dims, (weight, bias) = ctx.meta, ctx.dims, ctx.params
        names = [meta["prefix"] + "final_layer.weight", meta["prefix"] + "final_layer.bias"]
        ws = Workspace.get(lib.mmae_convnext_tail_workspace_bytes(*dims), dout.device)
        dout = dout.contiguous().float()
        dx = torch.empty((dims[0] * dims[1] * dims[2] * dims[3] * dims[3], dims[4]), dtype=torch.float32, device=dout.device)
        L.check(lib.mmae_convnext_tail_backward(dout.data_ptr(), *dims, meta["H"], meta["W"], weight.data_ptr(),
                                                _grad_ptr(meta["arena"], names[0]), _grad_ptr(meta["arena"], names[1]),
                                                dx.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_convnext_tail_backward")
        return (dx, None) + tuple(_report(meta, names, [weight, bias]))


SEGMENTER_TAIL_PARAM_NAMES = ["decoder_norm.weight", "decoder_norm.bias", "patch_proj.weight", "classes_proj.weight",
                              "mask_norm.weight", "mask_norm.bias"]


class SegmenterProjFunction(torch.autograd.Function):
    """Token gather + proj_dec + class tokens of SegmenterMaskTransformerAdapter.forward (multimae/output_adapters.py:
    454-458): encoder tokens [B, N, D] -> the fp32 sequence [B, n + K, E], patch tokens first (mmae_segmenter_proj_*).

    args: enc, meta, proj_dec.weight, proj_dec.bias, cls_emb.  meta: arena, prefix, on_grads_ready, save, n (tokens per
    task), starts (first token of each main task)."""

    @staticmethod
    def forward(ctx, enc, meta, weight, bias, cls_emb):
        _require_cuda(enc, "SegmenterMaskTransformerAdapter")
        lib = L.lib()
        enc = enc.contiguous().float()
        B, N, D = enc.shape
        n, starts, E, K = meta["n"], list(meta["starts"]), weight.shape[0], cls_emb.shape[1]
        arr = (ctypes.c_int * len(starts))(*starts)
        saved, saved_ptr, ws_ptr = _saved_and_ws(meta, lib.mmae_segmenter_proj_saved_bytes(B, n, D * len(starts), E),
                                                 lib.mmae_segmenter_proj_workspace_bytes(B, n, D * len(starts), E), enc.device)
        out = torch.empty((B, n + K, E), dtype=torch.float32, device=enc.device)
        L.check(lib.mmae_segmenter_proj_forward(enc.data_ptr(), B, N, D, n, len(starts), arr, E, K, weight.data_ptr(),
                                                bias.data_ptr(), cls_emb.data_ptr(), out.data_ptr(), saved_ptr, ws_ptr,
                                                L.current_stream()), "mmae_segmenter_proj_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, (B, N, D), (weight, bias, cls_emb)
            ctx.save_for_backward(saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        (saved,) = ctx.saved_tensors
        meta, (weight, bias, cls_emb) = ctx.meta, ctx.params
        B, N, D = ctx.dims
        n, starts, E, K = meta["n"], list(meta["starts"]), weight.shape[0], cls_emb.shape[1]
        arr = (ctypes.c_int * len(starts))(*starts)
        names = [meta["prefix"] + k for k in ("proj_dec.weight", "proj_dec.bias", "cls_emb")]
        ws = Workspace.get(lib.mmae_segmenter_proj_workspace_bytes(B, n, D * len(starts), E), dout.device)
        dout = dout.contiguous().float()
        denc = torch.empty((B, N, D), dtype=torch.float32, device=dout.device)
        L.check(lib.mmae_segmenter_proj_backward(dout.data_ptr(), B, N, D, n, len(starts), arr, E, K, weight.data_ptr(),
                                                 *[_grad_ptr(meta["arena"], k) for k in names], denc.data_ptr(),
                                                 saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_segmenter_proj_backward")
        return (denc, None) + tuple(_report(meta, names, [weight, bias, cls_emb]))


class SegmenterTailFunction(torch.autograd.Function):
    """Everything after the blocks of SegmenterMaskTransformerAdapter.forward (multimae/output_adapters.py:463-476):
    decoder_norm, patch_proj / classes_proj, the fused cosine mask + class LayerNorm, bilinear upsample: [B, n + K, E] ->
    [B, K, H, W] fp32 (mmae_segmenter_tail_*).  args: x, meta (plus B, nh, nw, num_classes, H, W, eps_dec, eps_mask), then
    the 6 SEGMENTER_TAIL_PARAM_NAMES tensors - the order of the entry points' pointer arrays."""

    @staticmethod
    def forward(ctx, x, meta, *params):
        _require_cuda(x, "SegmenterMaskTransformerAdapter")
        lib = L.lib()
        x = x.contiguous().float()
        K, H, W = meta["num_classes"], meta["H"], meta["W"]
        dims = (meta["B"], meta["nh"], meta["nw"], x.shape[2], K)
        saved, saved_ptr, ws_ptr = _saved_and_ws(meta, lib.mmae_segmenter_tail_saved_bytes(*dims),
                                                 lib.mmae_segmenter_tail_workspace_bytes(*dims), x.device)
        out = torch.empty((meta["B"], K, H, W), dtype=torch.float32, device=x.device)
        prm = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        L.check(lib.mmae_segmenter_tail_forward(x.data_ptr(), *dims, H, W, float(meta["eps_dec"]), float(meta["eps_mask"]), prm,
                                                out.data_ptr(), saved_ptr, ws_ptr, L.current_stream()),
                "mmae_segmenter_tail_forward")
        if saved is not None:
            ctx.meta, ctx.dims, ctx.params = meta, dims, params
            ctx.save_for_backward(x, saved)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.lib()
        x, saved = ctx.saved_tensors
        meta, dims, params = ctx.meta, ctx.dims, ctx.params
        names = [meta["prefix"] + k for k in SEGMENTER_TAIL_PARAM_NAMES]
        ws = Workspace.get(lib.mmae_segmenter_tail_workspace_bytes(*dims), dout.device)
        dout = dout.contiguous().float()
        dx = torch.empty_like(x)
        prm = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        grd = (ctypes.c_void_p * len(names))(*[_grad_ptr(meta["arena"], k) for k in names])
        L.check(lib.mmae_segmenter_tail_backward(x.data_ptr(), dout.data_ptr(), dx.data_ptr(), *dims, meta["H"], meta["W"],
                                                 prm, grd, saved.data_ptr(), ws.data_ptr(), L.current_stream()),
                "mmae_segmenter_tail_backward")
        return (dx, None) + tuple(_report(meta, names, params))


# ---------------------------------------------------------------------------------------------------------------------
# masked losses
# ---------------------------------------------------------------------------------------------------------------------
class MaskedLossFunction(torch.autograd.Function):
    """multimae/criterion.py losses; kind 0 = MSE, 1 = L1, 2 = cross-entropy."""

    @staticmethod
    def forward(ctx, pred, target, mask, kind, norm_pix, scale, label_smoothing):
        _require_cuda(pred, "criterion")
        lib = L.lib()
        pred = pred.contiguous().float()
        B, C, H, W = pred.shape
        if kind == 2:
            target = target.contiguous().long()
        else:
            target = target.contiguous().float()
        if mask is not None:
            mask = mask.contiguous().long()
        ws = torch.empty(2 * B, dtype=torch.float32, device=pred.device)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        L.check(lib.mmae_masked_loss_forward(kind, int(norm_pix), float(label_smoothing), pred.data_ptr(),
                                             target.data_ptr(), L.ptr(mask), B, C, H, W, scale, ws.data_ptr(),
                                             loss.data_ptr(), L.current_stream()), "mmae_masked_loss_forward")
        ctx.cfg = (kind, int(norm_pix), scale, float(label_smoothing))
        ctx.save_for_backward(pred, target, mask, ws)
        return loss

    @staticmethod
    def backward(ctx, gout):
        lib = L.lib()
        pred, target, mask, ws = ctx.saved_tensors
        kind, norm_pix, scale, smoothing = ctx.cfg
        B, C, H, W = pred.shape
        gout = gout.contiguous().float()
        dpred = torch.empty_like(pred)
        L.check(lib.mmae_masked_loss_backward(kind, norm_pix, smoothing, pred.data_ptr(), target.data_ptr(), L.ptr(mask),
                                              B, C, H, W, scale, ws.data_ptr(), gout.data_ptr(), dpred.data_ptr(),
                                              L.current_stream()), "mmae_masked_loss_backward")
        return dpred, None, None, None, None, None, None


# ---------------------------------------------------------------------------------------------------------------------
# mask sampler (no autograd)
# ---------------------------------------------------------------------------------------------------------------------
def sample_masks(shares, noise_task, noise_all, tokens_per_task, num_encoded):
    """Pure function of the random draws -> (mask_all [B,total] int64, ids_keep, ids_restore); one kernel launch."""
    _require_cuda(noise_all, "generate_random_masks")
    B, total = noise_all.shape
    dev = noise_all.device
    shares = shares.to(device=dev, dtype=torch.float32).contiguous()
    noise_task = noise_task.contiguous().float()
    noise_all = noise_all.contiguous().float()
    masks = torch.empty((B, total), dtype=torch.int64, device=dev)
    ids_keep = torch.empty((B, num_encoded), dtype=torch.int64, device=dev)
    ids_restore = torch.empty((B, total), dtype=torch.int64, device=dev)
    arr = (ctypes.c_int * len(tokens_per_task))(*tokens_per_task)
    L.check(L.lib().mmae_sample_masks(shares.data_ptr(), noise_task.data_ptr(), noise_all.data_ptr(), B,
                                      len(tokens_per_task), arr, num_encoded, masks.data_ptr(), ids_keep.data_ptr(),
                                      ids_restore.data_ptr(), L.current_stream()), "mmae_sample_masks")
    return masks, ids_keep, ids_restore


def standardize_depth(depth, lo_frac=0.1, hi_frac=0.9, eps=1e-6, out=None, return_stats=False):
    """Truncated depth standardisation of train_one_epoch (run_pretraining_multimae.py:487-492) in one kernel launch.

    depth [B, ...] fp32 on the device -> (depth - mean_b) / sqrt(var_b + eps), mean_b / var_b (unbiased) taken over the
    values of sample b whose rank lies in [int(lo_frac n), int(hi_frac n)) — the reference's sort + slice.  `out` may be
    `depth` itself.  With return_stats also returns the [B, 2] tensor of (mean, var)."""
    _require_cuda(depth, "standardize_depth")
    if depth.dtype != torch.float32:
        raise TypeError("standardize_depth: fp32 depth maps expected, got %s" % depth.dtype)
    x = depth.contiguous()
    B = x.shape[0]
    n = x[0].numel()
    lo, hi = int(lo_frac * n), int(hi_frac * n)           # the reference's own host-side expressions (:490)
    if out is None:
        out = torch.empty_like(x)
    elif out.shape != x.shape or out.dtype != torch.float32 or not out.is_contiguous() or out.device != x.device:
        raise ValueError("standardize_depth: `out` must be a contiguous fp32 tensor of the input's shape on its device")
    stats = torch.empty((B, 2), dtype=torch.float32, device=x.device) if return_stats else None
    L.check(L.lib().mmae_standardize_depth(x.data_ptr(), out.data_ptr(), B, n, lo, hi, float(eps), L.ptr(stats),
                                           L.current_stream()), "mmae_standardize_depth")
    return (out, stats) if return_stats else out


def grad_unscale_norm(flat, inv_scale=1.0, post_scale=1.0, inv_scale_tensor=None):
    """In-place flat *= inv_scale*post_scale; returns (norm tensor [1], out2 = [sum_sq, found_inf])."""
    _require_cuda(flat, "grad_unscale_norm")
    out2 = torch.empty(2, dtype=torch.float32, device=flat.device)
    norm = torch.empty((), dtype=torch.float32, device=flat.device)
    L.check(L.lib().mmae_grad_unscale_norm(flat.data_ptr(), flat.numel(), L.ptr(inv_scale_tensor), float(inv_scale),
                                           float(post_scale), out2.data_ptr(), norm.data_ptr(), L.current_stream()),
            "mmae_grad_unscale_norm")
    return norm, out2


def adamw_step(params, grads, exp_avg, exp_avg_sq, lr, betas, eps, weight_decay, step, found_inf=None, dyn=None):
    L.check(L.lib().mmae_adamw_step(params.data_ptr(), grads.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                    params.numel(), float(lr), float(betas[0]), float(betas[1]), float(eps),
                                    float(weight_decay), max(int(step), 1), L.ptr(found_inf), L.ptr(dyn),
                                    L.current_stream()), "mmae_adamw_step")


def adamw_step_groups(segments, count, lrs, weight_decays, betas, eps, step, found_inf=None):
    """One grouped AdamW step: `segments` a ctypes array of L.AdamwSegment (its first `count` entries are used), `lrs` /
    `weight_decays` ctypes double arrays with one entry per parameter group, `step` the device step counter (float32 [1])."""
    L.check(L.lib().mmae_adamw_step_groups(segments, count, lrs, weight_decays, len(lrs), float(betas[0]), float(betas[1]),
                                           float(eps), L.ptr(found_inf), step.data_ptr(), L.current_stream()),
            "mmae_adamw_step_groups")

