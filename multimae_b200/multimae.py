"""MultiMAE / MultiViT with the reference's module API (multimae/multimae.py), executing on sm_90a (H100) kernels.

Same constructor signature, parameter names / shapes (state_dict schema of SURVEY.md §A.1), factories registered under
the same names, and the same `forward` contract — `(preds, task_masks)` — so run_pretraining_multimae.py can drive it
unchanged.  What differs is the execution plan: gather-first patch embedding, one mask-sampler kernel,
fused transformer blocks, fused decoder head/tail, gradients accumulated into one flat arena.
"""
import itertools
import os
import math
import weakref
from collections import OrderedDict
from functools import partial
from typing import Dict, List, Optional, Union

import torch
from torch import nn
from torch.distributions.dirichlet import Dirichlet

from . import _lib as L
from . import functional as Fn
from .multimae_utils import Block, trunc_normal_
from .output_adapters import SpatialOutputAdapter

try:  # the reference's timm-style registry, when the reference tree is importable (drop-in overlay); else a local one
    from utils.registry import register_model  # type: ignore
except Exception:  # noqa: BLE001
    _LOCAL_REGISTRY = {}

    def register_model(fn):
        _LOCAL_REGISTRY[fn.__name__] = fn
        return fn

__all__ = ["pretrain_multimae_base", "pretrain_multimae_large", "multivit_base", "multivit_large"]

# Set by the overlay launcher: a model driven by the unchanged reference script makes its parameters' .grad alias the flat
# gradient arena on its first training forward, so that the script's scaler (which only sees model.parameters()) takes the
# one-pass unscale / norm path instead of ~344 per-tensor launches, and autograd does not clone 98 M gradients per step.
AUTO_OWN_GRADIENTS = False
# every MultiMAE / MultiViT alive: GroupedFlatAdamW finds the model that owns the parameters it is given here
_LIVE_MODELS = weakref.WeakSet()


def live_models():
    return list(_LIVE_MODELS)


# one GEMM for the proj_context Linears of all half-precision output adapters (MultiMAE._project_contexts); 0: one per adapter
SHARED_CONTEXT_PROJECTION = os.environ.get("MMAE_SHARED_CTX", "1") != "0"


def _build_layout(adapters, x):
    """EmbedLayout + per-task metadata for the ordered (name, adapter, tensor) triples."""
    layout = L.EmbedLayout()
    layout.num_tasks = len(adapters)
    if layout.num_tasks > L.MAX_TASKS:
        raise L.MmaeError("multimae_b200: at most %d input modalities" % L.MAX_TASKS)
    tok, k = 0, 0
    for t, (name, ad) in enumerate(adapters):
        nh, nw = ad.grid(x[name])
        assert ad.P_H == ad.P_W, "multimae_b200: square patches only"
        layout.grid_h[t], layout.grid_w[t] = nh, nw
        layout.tok_offset[t], layout.k_offset[t] = tok, k
        layout.patch[t] = ad.P_H
        layout.channels[t] = ad.embed_channels()
        layout.is_semseg[t] = 1 if ad.is_semseg else 0
        layout.num_classes[t] = ad.num_classes if ad.is_semseg else 0
        tok += nh * nw
        k += ad.embed_channels() * ad.P_H * ad.P_W
    layout.tok_offset[layout.num_tasks] = tok
    layout.k_offset[layout.num_tasks] = k
    return layout


def _embed(adapters, x, ids_keep, ids_restore, global_tokens, arena, prefix_of, on_grads_ready=None):
    """Gather-first embedding of the tokens listed in ids_keep (+ global tokens appended last).  A frozen position table
    enters as its cached resized rows; a trainable one (learnable_pos_emb=True / sincos_pos_emb=False) as an autograd input
    of EmbedFunction, resized on the device every call (ids_restore then locates each patch's token for its gradient)."""
    layout = _build_layout(adapters, x)
    names, tensors, pos, tables, pos_names = [], [], [], [], []
    for t, (name, ad) in enumerate(adapters):
        pre = prefix_of(name)
        cemb = ad.class_emb.weight if ad.is_semseg else None
        names.append((pre + "proj.weight", pre + "proj.bias", pre + "class_emb.weight" if ad.is_semseg else None))
        tensors += [x[name], ad.proj.weight, ad.proj.bias, cemb]
        if ad.pos_emb.requires_grad:
            pos.append(None)
            tables.append(ad.pos_emb)
            pos_names.append(pre + "pos_emb")
        else:
            pos.append(ad._resized_pos(layout.grid_h[t], layout.grid_w[t], ad.pos_mode))
            tables.append(None)
            pos_names.append(None)
    meta = dict(layout=layout, arena=arena, names=names, pos=pos, on_grads_ready=on_grads_ready)
    if not any(n is not None for n in pos_names):
        return Fn.EmbedFunction.apply(meta, ids_keep, *tensors, global_tokens)
    meta.update(ids_restore=ids_restore.contiguous(), pos_names=pos_names, pos_modes=[L.POS_MODES[ad.pos_mode] for _, ad in adapters])
    return Fn.EmbedFunction.apply(meta, ids_keep, *tensors, global_tokens, *tables)


def embed_all_patches(adapter, x):
    """Stand-alone input-adapter forward: every patch of one modality -> [B, N, D] (reference adapter.forward)."""
    Fn._require_cuda(x, "input adapter")
    nh, nw = adapter.grid(x)
    B = x.shape[0]
    ids = torch.arange(nh * nw, device=x.device).unsqueeze(0).expand(B, -1).contiguous()
    named = [(n, p) for n, p in adapter.named_parameters() if p.requires_grad]
    dummy = torch.zeros(1, 0, adapter.dim_tokens, device=x.device, requires_grad=False)
    arena = Fn.GradArena(named + [("global_tokens", dummy)], x.device)
    return _embed([("x", adapter)], {"x": x}, ids, ids, dummy, arena, lambda name: "")   # every patch kept, in order


class MultiMAE(nn.Module):
    """MultiMAE: Multi-task Multi-modal Masked Autoencoder (performs masking in its forward pass)."""

    def __init__(self, input_adapters: Dict[str, nn.Module], output_adapters: Optional[Dict[str, nn.Module]],
                 num_global_tokens: int = 1, dim_tokens: int = 768, depth: int = 12, num_heads: int = 12,
                 mlp_ratio: float = 4.0, qkv_bias: bool = True, drop_rate: float = 0.0, attn_drop_rate: float = 0.0,
                 drop_path_rate: float = 0.0, norm_layer: nn.Module = partial(nn.LayerNorm, eps=1e-6)):
        super().__init__()
        for adapter in input_adapters.values():
            adapter.init(dim_tokens=dim_tokens)
        self.input_adapters = nn.ModuleDict(input_adapters)
        if output_adapters is not None:
            for adapter in output_adapters.values():
                adapter.init(dim_tokens_enc=dim_tokens)
            self.output_adapters = nn.ModuleDict(output_adapters)
        else:
            self.output_adapters = None

        self.num_global_tokens = num_global_tokens
        self.global_tokens = nn.Parameter(torch.zeros(1, num_global_tokens, dim_tokens))
        trunc_normal_(self.global_tokens, std=0.02)

        dpr = [v.item() for v in torch.linspace(0, drop_path_rate, depth)]
        self.encoder = nn.Sequential(*[
            Block(dim=dim_tokens, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, drop=drop_rate,
                  attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer) for i in range(depth)])

        self._init_all_weights()
        self._arena = None
        self._grad_callback = None
        self.external_shares = None
        self.device_shares = False                 # draw the Dirichlet task shares on the device (graph capture)
        self._alphas_dev = None
        # task decoders on concurrent CUDA streams (MMAE_DECODER_STREAMS=0 runs them one after the other)
        self.decoder_streams = os.environ.get("MMAE_DECODER_STREAMS", "1") != "0"
        self._dec_streams = None
        _LIVE_MODELS.add(self)

    def draw_task_shares(self, B, n_tasks, alphas=1.0, sample_tasks_uniformly=False):
        """Host-side Dirichlet draw of generate_random_masks (multimae/multimae.py:182-187) as a separate step."""
        alphas = [alphas] * n_tasks if isinstance(alphas, float) else alphas
        if sample_tasks_uniformly:
            return Dirichlet(self.sample_alphas(B, n_tasks, alphas=alphas)).sample()
        return Dirichlet(torch.Tensor(alphas)).sample((B,))

    # ------------------------------------------------------------------------------------------------------------
    # initialisation, same scheme as multimae/multimae.py:100-125
    # ------------------------------------------------------------------------------------------------------------
    def _init_all_weights(self):
        for name, m in self.named_modules():
            if isinstance(m, nn.Linear):
                fan_out, fan_in = m.weight.shape
                if "qkv" in name:       # q, k, v initialised as three separate square-ish matrices
                    fan_out //= 3
                elif "kv" in name:
                    fan_out //= 2
                bound = math.sqrt(6.0 / float(fan_out + fan_in))
                nn.init.uniform_(m.weight, -bound, bound)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.LayerNorm):
                nn.init.constant_(m.bias, 0)
                nn.init.constant_(m.weight, 1.0)
            elif isinstance(m, nn.Conv2d) and ".proj" in name:
                w = m.weight.data
                nn.init.xavier_uniform_(w.view([w.shape[0], -1]))   # like nn.Linear (MAE)

    def get_num_layers(self):
        return len(self.encoder)

    @torch.jit.ignore
    def no_weight_decay(self):
        no_wd = {"global_tokens"}
        for group, adapters in (("input_adapters", self.input_adapters), ("output_adapters", self.output_adapters or {})):
            for task, adapter in adapters.items():
                if hasattr(adapter, "no_weight_decay"):
                    no_wd |= {f"{group}.{task}.{n}" for n in adapter.no_weight_decay()}
        return no_wd

    # ------------------------------------------------------------------------------------------------------------
    # gradient arena (flat fp32 buffer the kernels accumulate into)
    # ------------------------------------------------------------------------------------------------------------
    def grad_arena(self, device=None):
        device = device if device is not None else self.global_tokens.device
        if self._arena is None or self._arena.flat.device != device:
            named = [(n, p) for n, p in self.named_parameters() if p.requires_grad]
            # proj_context weights (then biases) of the output adapters back to back: their gradient slots - and, once
            # FlatAdamW lays parameters / moments / the bf16 mirror out like the arena, the operands themselves - form ONE
            # [sum Dd, D_enc] matrix that the shared context projection (SharedContextFunction) uses in place
            for suffix in (".proj_context.weight", ".proj_context.bias"):
                pc = [i for i, (n, _) in enumerate(named) if n.startswith("output_adapters.") and n.endswith(suffix)]
                if len(pc) > 1:
                    moved = [named[i] for i in pc]
                    rest = [e for i, e in enumerate(named) if i not in set(pc)]
                    named = rest[:pc[0]] + moved + rest[pc[0]:]
            self._arena = Fn.GradArena(named, device)
            self._bind()
        return self._arena

    def set_grad_callback(self, fn):
        """fn(names) is called from backward as soon as the gradients of `names` are complete in the arena."""
        self._grad_callback = fn
        if self._arena is not None:
            self._bind()

    def _bind(self):
        for i, blk in enumerate(self.encoder):
            blk.bind(self._arena, "encoder.%d." % i, self._grad_callback)
        if self.output_adapters is not None:
            for key, ad in self.output_adapters.items():
                if hasattr(ad, "bind"):
                    ad.bind(self._arena, "output_adapters.%s." % key, self._grad_callback)

    def own_gradients(self, owned=True):
        """`owned`: every p.grad permanently aliases its arena view (flat all-reduce / fused optimizer)."""
        arena = self.grad_arena()
        arena.owned = owned
        if owned:
            for n, p in self.named_parameters():
                if p.requires_grad:
                    p.grad = arena.views[n]
        return arena

    # ------------------------------------------------------------------------------------------------------------
    # mask sampling (multimae/multimae.py:148-218)
    # ------------------------------------------------------------------------------------------------------------
    def sample_alphas(self, B: int, n_tasks: int, alphas: float = 1.0, eps: float = 1e-5):
        choices = torch.Tensor([list(i) for i in itertools.product([0, 1], repeat=n_tasks)][1:])
        pick = torch.randint(0, len(choices), (B,))
        return torch.index_select(choices, 0, pick) * torch.tensor(alphas) + eps

    def generate_random_masks(self, input_tokens: Dict[str, torch.Tensor], num_encoded_tokens: int,
                              alphas: Union[float, List[float]] = 1.0, sample_tasks_uniformly: bool = False):
        """Dirichlet task shares on the host (as the reference), uniform noise with torch's device generator in the
        reference's consumption order, then ONE kernel for everything else."""
        first = list(input_tokens.values())[0]
        B, device = first.shape[0], first.device
        alphas = [alphas] * len(input_tokens) if isinstance(alphas, float) else alphas
        if self.external_shares is not None:
            # CUDA-graph mode with host draws: the Dirichlet draw is made outside the captured region and copied into
            # this static device buffer before every replay
            shares = self.external_shares
        elif self.device_shares and first.is_cuda and not sample_tasks_uniformly:
            # CUDA-graph mode (train_step.TrainStep.capture): the same Dirichlet(alphas) draw with the device generator,
            # so the replayed step needs no host -> device traffic at all
            key = (tuple(float(a) for a in alphas), device)
            if self._alphas_dev is None or self._alphas_dev[0] != key:      # created outside any capture (warm-up step)
                self._alphas_dev = (key, torch.tensor(key[0], dtype=torch.float32, device=device))
            shares = Dirichlet(self._alphas_dev[1], validate_args=False).sample((B,))
        elif sample_tasks_uniformly:
            shares = Dirichlet(self.sample_alphas(B, len(input_tokens), alphas=alphas)).sample()
        else:
            shares = Dirichlet(torch.Tensor(alphas)).sample((B,))
        counts = [t.shape[1] for t in input_tokens.values()]
        noise_task = torch.cat([torch.rand(B, n, device=device) for n in counts], dim=1)
        noise_all = torch.rand(B, sum(counts), device=device)
        mask_all, ids_keep, ids_restore = Fn.sample_masks(shares, noise_task, noise_all, counts, num_encoded_tokens)
        task_masks = dict(zip(input_tokens.keys(), torch.split(mask_all, counts, dim=1)))
        return task_masks, ids_keep, ids_restore

    @staticmethod
    def make_mask(N_H, N_W, xy_idxs, full_tasks=[], indicate_visible=True, flatten=True, device="cuda"):
        """Masks for each task from lists of un-masked (x, y) coordinates (multimae/multimae.py:220-248)."""
        masks = {}
        for k, v in xy_idxs.items():
            m = torch.ones(N_H, N_W, device=device)
            idx = torch.as_tensor(v, dtype=torch.long)
            if len(idx) > 0:
                m[idx[:, 1], idx[:, 0]] = 0
            if k in full_tasks:
                m[:] = 0
            masks[k] = m
        if not indicate_visible:
            masks = {k: 1 - v for k, v in masks.items()}
        if flatten:
            masks = {k: v.flatten().unsqueeze(0) for k, v in masks.items()}
        return masks

    def generate_input_info(self, input_task_tokens, image_size):
        info = OrderedDict()
        info["tasks"] = {}
        i = 0
        for domain, tensor in input_task_tokens.items():
            n = tensor.shape[1]
            info["tasks"][domain] = {"num_tokens": n, "has_2d_posemb": True, "start_idx": i, "end_idx": i + n}
            i += n
        info["image_size"] = image_size
        info["num_task_tokens"] = i
        info["num_global_tokens"] = self.num_global_tokens
        return info

    # ------------------------------------------------------------------------------------------------------------
    def _prepare(self, x):
        x = {"rgb": x} if isinstance(x, torch.Tensor) else x
        if "rgb" in x:
            B, _, H, W = x["rgb"].shape
        elif "semseg" in x:
            B, H, W = x["semseg"].shape
            H *= self.input_adapters["semseg"].stride_level
            W *= self.input_adapters["semseg"].stride_level
        else:
            B, _, H, W = list(x.values())[0].shape
        adapters = [(d, self.input_adapters[d]) for d in x if d in self.input_adapters]
        if not adapters:
            raise ValueError("no input modality matches the model's input adapters")
        dev = x[adapters[0][0]].device
        Fn._require_cuda(x[adapters[0][0]], "MultiMAE.forward")
        # token placeholders: only B / N_t / device are read downstream (the tokens are never materialised)
        placeholders = OrderedDict()
        for name, ad in adapters:
            nh, nw = ad.grid(x[name])
            placeholders[name] = torch.empty((B, nh * nw, 0), device=dev)
        return x, adapters, placeholders, B, H, W, dev

    def forward(self, x: Union[Dict[str, torch.Tensor], torch.Tensor], mask_inputs: bool = True,
                task_masks: Dict[str, torch.Tensor] = None, num_encoded_tokens: int = 128,
                alphas: Union[float, List[float]] = 1.0, sample_tasks_uniformly: bool = False,
                fp32_output_adapters: List[str] = []):
        Fn.fresh_mirrors()                                    # bf16 weight twins follow any torch-side parameter change
        Fn.sync_deterministic()
        x, adapters, placeholders, B, H, W, dev = self._prepare(x)
        input_info = self.generate_input_info(input_task_tokens=placeholders, image_size=(H, W))
        total = input_info["num_task_tokens"]
        if not mask_inputs:
            num_encoded_tokens = total
        elif num_encoded_tokens is None:
            num_encoded_tokens = self.num_encoded_tokens

        if task_masks is None:
            task_masks, ids_keep, ids_restore = self.generate_random_masks(
                placeholders, num_encoded_tokens, alphas=alphas, sample_tasks_uniformly=sample_tasks_uniformly)
        else:
            # fixed masks: visible tokens first, original order kept (stable).  The reference derives ONE count from
            # the whole batch (multimae/multimae.py:338, correct only for B=1); here every sample must expose the same
            # number of visible tokens and that per-sample count is used.
            mask_all = torch.cat([task_masks[t].to(dev) for t in placeholders], dim=1)
            ids_shuffle = torch.argsort(mask_all, dim=1, stable=True)
            ids_restore = torch.argsort(ids_shuffle, dim=1, stable=True)
            n_vis = (mask_all == 0).sum(dim=1)
            if not bool((n_vis == n_vis[0]).all()):
                raise ValueError("multimae_b200: fixed task_masks must keep the same number of visible tokens per sample")
            ids_keep = ids_shuffle[:, :int(n_vis[0])]

        arena = self.grad_arena(dev)
        if torch.is_grad_enabled() and self.training:
            if AUTO_OWN_GRADIENTS and not arena.owned:
                self.own_gradients(True)
            arena.begin_step()
        seq = _embed(adapters, x, ids_keep, ids_restore, self.global_tokens, arena, lambda d: "input_adapters.%s." % d,
                     self._grad_callback)
        encoder_tokens = Fn.block_stack(self.encoder, seq)
        if self.output_adapters is None:
            return encoder_tokens, task_masks

        preds = self._decode(encoder_tokens, input_info, ids_keep, ids_restore, fp32_output_adapters)
        return preds, task_masks

    def _project_contexts(self, encoder_tokens, domains):
        """One GEMM for the proj_context Linears (multimae/output_adapters.py:258) of the half-precision spatial adapters -
        they all project the same encoder output (multimae/multimae.py:357-366).  Returns {domain: shared_ctx dict} (empty
        when fewer than two adapters qualify or MMAE_SHARED_CTX=0)."""
        if not SHARED_CONTEXT_PROJECTION or self._arena is None:
            return {}
        group = []
        for d in domains:
            ad = self.output_adapters[d]
            if (isinstance(ad, SpatialOutputAdapter) and ad.use_xattn and ad.dim_tokens % 8 == 0
                    and ad.dim_tokens_enc == encoder_tokens.shape[-1] and ad._bound is not None
                    and ad._bound["arena"] is self._arena):
                group.append(d)
        if not 2 <= len(group) <= L.MAX_TASKS:
            return {}
        adapters = [self.output_adapters[d] for d in group]
        wb = []
        for ad in adapters:
            wb += [ad.proj_context.weight, ad.proj_context.bias]
        state = {}
        meta = dict(arena=self._arena, weight_names=["output_adapters.%s.proj_context.weight" % d for d in group],
                    on_grads_ready=self._grad_callback, state=state)
        ctx = Fn.SharedContextFunction.apply(encoder_tokens, meta, *wb)
        out, off = {}, 0
        for d, ad in zip(group, adapters):
            out[d] = dict(ctx=ctx, offset=off, ld=ctx.shape[1], state=state, enc_shape=tuple(encoder_tokens.shape))
            off += ad.dim_tokens
        return out

    def _decode(self, encoder_tokens, input_info, ids_keep, ids_restore, fp32_output_adapters=()):
        """The task decoders are independent of each other (multimae/multimae.py:372-381 runs them in a Python loop):
        on CUDA each runs on its own stream, forward and (through autograd's stream tracking) backward, so their
        1.3-wave GEMMs, phase-locked attention CTAs and element-wise tails fill each other's idle SMs."""
        domains = list(self.output_adapters)
        kw = dict(encoder_tokens=encoder_tokens, input_info=input_info, ids_keep=ids_keep, ids_restore=ids_restore)
        # adapters listed in fp32_output_adapters run in the fp32 tier (the reference calls them outside autocast,
        # multimae/multimae.py:367-377); custom adapter classes without the switch are called as the reference does
        fp32 = {d for d in (fp32_output_adapters or ()) if d in self.output_adapters}

        shared = self._project_contexts(encoder_tokens, [d for d in domains if d not in fp32])

        def run(d):
            if d in fp32:
                return self.output_adapters[d](fp32=True, **kw)
            if d in shared:
                return self.output_adapters[d](shared_ctx=shared[d], **kw)
            return self.output_adapters[d](**kw)

        if not (self.decoder_streams and encoder_tokens.is_cuda and len(domains) > 1):
            return {d: run(d) for d in domains}
        dev = encoder_tokens.device
        if self._dec_streams is None or len(self._dec_streams) != len(domains):
            self._dec_streams = [torch.cuda.Stream(device=dev) for _ in domains]
        main = torch.cuda.current_stream(dev)
        ready = main.record_event()
        if shared:                                    # allocated on this stream, read / written on the decoders' streams
            sh = next(iter(shared.values()))          # every entry carries the same projection tensor and state
            for st in self._dec_streams:
                sh["ctx"].record_stream(st)
                if sh["state"].get("dctx") is not None:
                    sh["state"]["dctx"].record_stream(st)
        preds = {}
        for d, st in zip(domains, self._dec_streams):
            st.wait_event(ready)
            with torch.cuda.stream(st):
                preds[d] = run(d)
        for d, st in zip(domains, self._dec_streams):
            main.wait_stream(st)
            preds[d].record_stream(main)              # allocated on the side stream, consumed (loss) on this one
        for t in (encoder_tokens, ids_keep, ids_restore):
            for st in self._dec_streams:
                t.record_stream(st)
        return preds


@register_model
def pretrain_multimae_base(input_adapters: Dict[str, nn.Module], output_adapters: Optional[Dict[str, nn.Module]], **kwargs):
    return MultiMAE(input_adapters=input_adapters, output_adapters=output_adapters, dim_tokens=768, depth=12, num_heads=12,
                    mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


@register_model
def pretrain_multimae_large(input_adapters: Dict[str, nn.Module], output_adapters: Optional[Dict[str, nn.Module]], **kwargs):
    return MultiMAE(input_adapters=input_adapters, output_adapters=output_adapters, dim_tokens=1024, depth=24,
                    num_heads=16, mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


class MultiViT(MultiMAE):
    """MultiMAE without masking (multimae/multimae.py:419-502): all tokens of all given modalities are encoded."""

    def process_input(self, x):
        x, adapters, placeholders, B, H, W, dev = self._prepare(x)
        input_info = self.generate_input_info(input_task_tokens=placeholders, image_size=(H, W))
        total = input_info["num_task_tokens"]
        ids = torch.arange(total, device=dev).unsqueeze(0).expand(B, -1).contiguous()
        arena = self.grad_arena(dev)
        if torch.is_grad_enabled() and self.training:
            if AUTO_OWN_GRADIENTS and not arena.owned:
                self.own_gradients(True)
            arena.begin_step()
        seq = _embed(adapters, x, ids, ids, self.global_tokens, arena, lambda d: "input_adapters.%s." % d,
                     self._grad_callback)                      # nothing masked: ids_restore is the identity, like ids
        return seq, input_info

    def forward(self, x, return_all_layers=False, **kwargs):
        Fn.fresh_mirrors()
        Fn.sync_deterministic()
        tokens, input_info = self.process_input(x)
        if not return_all_layers:
            encoder_tokens = Fn.block_stack(self.encoder, tokens)
        else:
            encoder_tokens = []
            for block in self.encoder:
                tokens = block(tokens)
                encoder_tokens.append(tokens)
        if self.output_adapters is None:
            return encoder_tokens
        return {domain: self.output_adapters[domain](encoder_tokens=encoder_tokens, input_info=input_info)
                for domain in self.output_adapters}


@register_model
def multivit_base(input_adapters: Dict[str, nn.Module], output_adapters: Optional[Dict[str, nn.Module]], **kwargs):
    return MultiViT(input_adapters=input_adapters, output_adapters=output_adapters, dim_tokens=768, depth=12, num_heads=12,
                    mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


@register_model
def multivit_large(input_adapters: Dict[str, nn.Module], output_adapters: Optional[Dict[str, nn.Module]], **kwargs):
    return MultiViT(input_adapters=input_adapters, output_adapters=output_adapters, dim_tokens=1024, depth=24,
                    num_heads=16, mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)
