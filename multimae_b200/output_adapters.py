"""Output adapters with the reference's constructor / state_dict / forward contract (multimae/output_adapters.py):

  SpatialOutputAdapter (:33-282) - the pre-training decoder, executed as DecoderHeadFunction -> Block x depth ->
                                   DecoderTailFunction;
  LinearOutputAdapter (:285-356) - the classification head of fine-tuning (run_finetuning_cls.py), one ClsHeadFunction;
  ConvNeXtAdapter (:481-573)     - the semantic-segmentation head of fine-tuning (run_finetuning_semseg.py), executed as
                                   ConvNeXtProjFunction -> ConvNeXtBlockFunction x depth -> ConvNeXtTailFunction.

  SegmenterMaskTransformerAdapter (:359-478) - the Segmenter head of the same script (--output_adapter segmenter),
                                   executed as SegmenterProjFunction -> Block x depth -> SegmenterTailFunction.

DPTOutputAdapter exists so that the fine-tuning scripts import; constructing it raises NotImplementedError."""
import math
from functools import partial
from typing import Dict, Iterable, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import functional as Fn
from .input_adapters import _PosEmbCache
from .multimae_utils import Block, CrossAttention, Mlp, build_2d_sincos_posemb, pair, trunc_normal_


class SpatialOutputAdapter(nn.Module, _PosEmbCache):
    """Cross-attention adapter for spatial outputs, like images or feature maps."""

    def __init__(self, num_channels: int, stride_level: int, patch_size_full: Union[int, Tuple[int, int]],
                 dim_tokens_enc: Optional[int] = None, dim_tokens: int = 256, depth: int = 0,
                 learnable_pos_emb: int = False, image_size: Union[int, Tuple[int]] = 224, mlp_ratio: int = 4.0,
                 num_heads: int = 8, qkv_bias: bool = True, drop_rate: float = 0.0, attn_drop_rate: float = 0.0,
                 drop_path_rate: float = 0.0, norm_layer: nn.Module = partial(nn.LayerNorm, eps=1e-6),
                 use_task_queries: bool = True, task: Optional[str] = None, context_tasks: Optional[list] = None,
                 use_xattn: bool = True):
        super().__init__()
        self.num_channels = num_channels
        self.stride_level = stride_level
        self.patch_size_full = pair(patch_size_full)
        self.dim_tokens_enc = dim_tokens_enc
        self.dim_tokens = dim_tokens
        self.learnable_pos_emb = learnable_pos_emb
        self.image_size = pair(image_size)
        self.use_task_queries = use_task_queries
        self.task = task
        self.use_xattn = use_xattn
        self.num_heads = num_heads
        self.P_H = max(1, self.patch_size_full[0] // stride_level)
        self.P_W = max(1, self.patch_size_full[1] // stride_level)
        assert self.P_H == self.P_W, "multimae_b200: square patches only"

        self.task_embeddings = None
        if context_tasks is not None:
            self.task_embeddings = nn.ParameterDict(
                {t: nn.Parameter(torch.zeros(1, 1, self.dim_tokens)) for t in context_tasks})
            for emb in self.task_embeddings.values():
                trunc_normal_(emb, std=0.02)

        self.mask_token = nn.Parameter(torch.zeros(1, 1, self.dim_tokens))

        h_posemb = self.image_size[0] // (self.stride_level * self.P_H)
        w_posemb = self.image_size[1] // (self.stride_level * self.P_W)
        if not self.learnable_pos_emb:
            self.pos_emb = nn.Parameter(build_2d_sincos_posemb(h=h_posemb, w=w_posemb, embed_dim=self.dim_tokens),
                                        requires_grad=False)
        else:
            self.pos_emb = nn.Parameter(torch.zeros(1, h_posemb, w_posemb, self.dim_tokens))
            trunc_normal_(self.pos_emb, std=0.02)

        if self.use_xattn:
            self.decoder = CrossAttention(dim=self.dim_tokens, num_heads=num_heads, qkv_bias=qkv_bias,
                                          attn_drop=attn_drop_rate, proj_drop=drop_rate)
            self.context_norm = norm_layer(self.dim_tokens)
            self.query_norm = norm_layer(self.dim_tokens)
            self.out_norm = norm_layer(self.dim_tokens)
            self.mlp_hidden = int(self.dim_tokens * mlp_ratio)
            self.mlp = Mlp(in_features=self.dim_tokens, hidden_features=self.mlp_hidden)

        if depth > 0:
            dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
            self.decoder_transformer = nn.Sequential(*[
                Block(dim=self.dim_tokens, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, drop=drop_rate,
                      attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer) for i in range(depth)])
        else:
            self.decoder_transformer = nn.Identity()

        self.dim_patch = self.num_channels * self.P_H * self.P_W
        self.out_proj = nn.Linear(self.dim_tokens, self.dim_patch)
        self._bound = None
        if self.dim_tokens_enc is not None:
            self.init(dim_tokens_enc=dim_tokens_enc)

    def init(self, dim_tokens_enc: int = 768):
        self.dim_tokens_enc = dim_tokens_enc
        self.proj_context = nn.Linear(self.dim_tokens_enc, self.dim_tokens)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_emb", "mask_token", "task_embeddings"}

    # ------------------------------------------------------------------------------------------------------------
    def bind(self, arena, prefix, on_grads_ready=None):
        self._bound = dict(arena=arena, prefix=prefix, on_grads_ready=on_grads_ready)
        if isinstance(self.decoder_transformer, nn.Sequential):
            for i, blk in enumerate(self.decoder_transformer):
                blk.bind(arena, "%sdecoder_transformer.%d." % (prefix, i), on_grads_ready)

    def _head_params(self):
        return (self.proj_context.weight, self.proj_context.bias, self.mask_token, self.context_norm.weight,
                self.context_norm.bias, self.query_norm.weight, self.query_norm.bias, self.out_norm.weight,
                self.out_norm.bias, self.decoder.q.weight, self.decoder.q.bias, self.decoder.kv.weight,
                self.decoder.kv.bias, self.decoder.proj.weight, self.decoder.proj.bias, self.mlp.fc1.weight,
                self.mlp.fc1.bias, self.mlp.fc2.weight, self.mlp.fc2.bias)

    def forward(self, encoder_tokens: torch.Tensor, input_info: Dict, ids_keep: torch.Tensor, ids_restore: torch.Tensor,
                fp32: bool = False, shared_ctx: Dict = None):
        """`fp32` (beyond the reference signature): run the whole adapter in the fp32 tier - what the reference does for the
        adapters listed in `fp32_output_adapters` by calling them outside autocast (multimae/multimae.py:367-377).
        `shared_ctx` (set by MultiMAE._decode): proj_context was already applied for all adapters in one GEMM
        (functional.SharedContextFunction); dict(ctx=[B*Nc, sum Dd] tensor, offset, ld, state, enc_shape)."""
        assert self.dim_tokens_enc is not None, "Need to call init(dim_tokens_enc) function first"
        if not self.use_xattn:
            raise NotImplementedError("multimae_b200: use_xattn=False is outside the pre-training hot path")
        if self.learnable_pos_emb:
            raise NotImplementedError("multimae_b200: learnable_pos_emb=True is outside the pre-training hot path")
        H, W = input_info["image_size"]
        nh = H // (self.stride_level * self.P_H)
        nw = W // (self.stride_level * self.P_W)
        tasks = list(input_info["tasks"].keys())
        task_names = list(tasks)
        task_embs = [self.task_embeddings[t] if (self.task_embeddings is not None and t in self.task_embeddings) else None
                     for t in tasks]
        if self.use_task_queries and self.task in tasks:
            # queries = this task's rows of the restored, embedded context (multimae/output_adapters.py:209-213)
            query_mode, own_task = 0, tasks.index(self.task)
        else:
            # queries = mask_token + pos_emb (+ this task's embedding when there is one) (:214-221): use_task_queries=False,
            # or a task that is reconstructed without being an input (e.g. --in_domains rgb --out_domains rgb-depth-semseg)
            query_mode, own_task = 1, -1
            if self.task_embeddings is not None and self.task in self.task_embeddings:
                if self.task in tasks:
                    own_task = tasks.index(self.task)
                else:                                        # an embedding that belongs to none of the given inputs
                    if len(tasks) >= Fn.L.MAX_TASKS:
                        raise Fn.L.MmaeError("multimae_b200: no free task slot for the query task embedding")
                    own_task = len(tasks)
                    task_names.append(self.task)
                    task_embs.append(self.task_embeddings[self.task])
        tok_offset = [input_info["tasks"][t]["start_idx"] for t in tasks] + [input_info["num_task_tokens"]]
        for t in tasks:
            assert input_info["tasks"][t]["num_tokens"] == nh * nw, "context tasks must share the adapter's patch grid"
        if self._bound is None or self._bound["arena"].flat.device != encoder_tokens.device:
            self.bind(Fn.GradArena([(n, p) for n, p in self.named_parameters() if p.requires_grad],
                                   encoder_tokens.device), "")
            self._own_arena = True
        if getattr(self, "_own_arena", False) and torch.is_grad_enabled():
            self._bound["arena"].zero_()
        head_meta = dict(self._bound, dim=self.dim_tokens, num_global=input_info.get("num_global_tokens", 0),
                         num_queries=nh * nw, tok_offset=tok_offset, own_task=own_task, query_mode=query_mode,
                         heads=self.num_heads, hidden=self.mlp_hidden, eps=self.query_norm.eps,
                         pos=self._resized_pos(nh, nw, "bilinear"), task_names=task_names, fp32=bool(fp32))
        head_params = self._head_params()
        head_in = encoder_tokens
        if shared_ctx is not None:
            assert not fp32, "the shared context projection is the half-precision tier"
            head_meta["shared"] = {k: shared_ctx[k] for k in ("offset", "ld", "state", "enc_shape")}
            head_in = shared_ctx["ctx"]
            head_params = (None,) + head_params[1:]          # proj_context.weight: used and differentiated by the shared GEMM
        x = Fn.DecoderHeadFunction.apply(head_in, head_meta, ids_keep, ids_restore, *head_params, *task_embs)
        if isinstance(self.decoder_transformer, nn.Sequential):
            x = Fn.block_stack(self.decoder_transformer, x, fp32=bool(fp32))
        else:
            x = self.decoder_transformer(x)
        tail_meta = dict(self._bound, nh=nh, nw=nw, channels=self.num_channels, patch=self.P_H, fp32=bool(fp32))
        return Fn.DecoderTailFunction.apply(x, tail_meta, self.out_proj.weight, self.out_proj.bias)


class LinearOutputAdapter(nn.Module):
    """Linear output adapter: head(norm(pool(encoder_tokens))), the pool being the mean over all tokens (global token
    included) or the last token (the global token).  Runs as one functional.ClsHeadFunction (mmae_clshead_*)."""

    def __init__(self, num_classes: int, dim_tokens_enc: Optional[int] = None, use_mean_pooling: bool = True,
                 norm_layer: nn.Module = partial(nn.LayerNorm, eps=1e-6), init_scale: float = 1.0):
        super().__init__()
        self.num_classes = num_classes
        self.dim_tokens_enc = dim_tokens_enc
        self.use_mean_pooling = use_mean_pooling
        self.norm_layer = norm_layer
        self.init_scale = init_scale
        self._bound = None
        if self.dim_tokens_enc is not None:
            self.init(dim_tokens_enc=dim_tokens_enc)

    def init(self, dim_tokens_enc: int = 768):
        """Build norm / head for encoder tokens of width dim_tokens_enc (called by MultiMAE.__init__).  A model that
        re-initialises all its modules afterwards (MultiMAE._init_all_weights, like the reference's
        multimae/multimae.py:100) overrides this trunc_normal / init_scale initialisation."""
        self._forbid_rebuild()
        self._bound = None
        self.dim_tokens_enc = dim_tokens_enc
        self.norm = self.norm_layer(self.dim_tokens_enc)
        assert isinstance(self.norm, nn.LayerNorm), "multimae_b200: norm_layer must build nn.LayerNorm"
        self.head = nn.Linear(dim_tokens_enc, self.num_classes) if self.num_classes > 0 else nn.Identity()
        self.apply(self._init_weights)
        if self.num_classes > 0:
            self.head.weight.data.mul_(self.init_scale)
            self.head.bias.data.mul_(self.init_scale)

    def _forbid_rebuild(self):
        if self._bound is not None and not getattr(self, "_own_arena", False):
            raise RuntimeError("LinearOutputAdapter: the head cannot be rebuilt once the model's gradient arena exists "
                               "(its gradient slots have the old shapes); reset the classifier before the first forward, "
                               "or build a new model")

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def get_classifier(self):
        return self.head

    def reset_classifier(self, num_classes, global_pool=''):
        """New head (and norm) for `num_classes`; raises once the model's gradient arena has been built."""
        self._forbid_rebuild()
        self.num_classes = num_classes
        self.init(dim_tokens_enc=self.dim_tokens_enc)

    def bind(self, arena, prefix, on_grads_ready=None):
        self._own_arena = False
        self._bound = dict(arena=arena, prefix=prefix, on_grads_ready=on_grads_ready)

    def forward(self, encoder_tokens: torch.Tensor, **kwargs):
        assert self.dim_tokens_enc is not None, "Need to call init(dim_tokens_enc) function first"
        if not torch.is_tensor(encoder_tokens):
            raise NotImplementedError("multimae_b200: LinearOutputAdapter takes the last layer's tokens "
                                      "(return_all_layers=False)")
        if self._bound is None or self._bound["arena"].flat.device != encoder_tokens.device:
            # stand-alone use (outside MultiMAE / MultiViT): private gradient arena, zeroed on every training forward
            self.bind(Fn.GradArena([(n, p) for n, p in self.named_parameters() if p.requires_grad],
                                   encoder_tokens.device), "")
            self._own_arena = True
        params = (self.norm.weight, self.norm.bias) + ((self.head.weight, self.head.bias) if self.num_classes > 0
                                                        else (None, None))
        save = torch.is_grad_enabled() and (encoder_tokens.requires_grad or
                                            any(p is not None and p.requires_grad for p in params))
        if self._own_arena and save:
            self._bound["arena"].zero_()
        meta = dict(self._bound, num_classes=self.num_classes, mean_pool=self.use_mean_pooling, eps=self.norm.eps,
                    save=save)
        return Fn.ClsHeadFunction.apply(encoder_tokens, meta, *params)


class ConvNeXtBlock(nn.Module):
    """ConvNeXt block (multimae/output_adapter_utils.py:19-57) as the adapter builds it: no layer scale (gamma None) and no
    stochastic depth.  x + pwconv2(GELU(pwconv1(LN(dwconv(x))))); executed by functional.ConvNeXtBlockFunction."""

    def __init__(self, dim):
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, 4 * dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(4 * dim, dim)
        self.gamma = None
        self.drop_path = nn.Identity()

    def _params(self):
        return (self.dwconv.weight, self.dwconv.bias, self.norm.weight, self.norm.bias, self.pwconv1.weight,
                self.pwconv1.bias, self.pwconv2.weight, self.pwconv2.bias)


class ConvNeXtAdapter(nn.Module):
    """Output adapter with ConvNeXt blocks for semantic segmentation: proj_dec of the main tasks' tokens, reshaped into a
    (nh*s) x (nw*s) map of embed_dim / preds_per_patch channels (s = sqrt(preds_per_patch)), `depth` ConvNeXt blocks, a 1x1
    conv to num_classes and a bilinear upsample to the image size.  Extra keyword arguments (stride_level, ...) are
    ignored, as by the reference.

    The kernels keep the map as a [pixels, channels] matrix whose LayerNorm needs embed_dim / preds_per_patch to be a
    multiple of 128 and at most 1024 (384 in every shipped semseg config); other widths raise here."""

    def __init__(self, num_classes, embed_dim: int = 6144, preds_per_patch: int = 16, main_tasks: Iterable[str] = ('rgb',),
                 patch_size: int = 16, depth: int = 4, interpolate_mode: str = 'bilinear', **kwargs):
        super().__init__()
        s = int(round(math.sqrt(preds_per_patch)))
        if preds_per_patch <= 0 or s * s != preds_per_patch:
            raise ValueError("ConvNeXtAdapter: preds_per_patch=%r must be a perfect square" % (preds_per_patch,))
        if embed_dim % preds_per_patch != 0:
            raise ValueError("ConvNeXtAdapter: embed_dim=%d is not divisible by preds_per_patch=%d"
                             % (embed_dim, preds_per_patch))
        class_dim = embed_dim // preds_per_patch
        if class_dim % 128 != 0 or class_dim > 1024:
            raise NotImplementedError(
                "ConvNeXtAdapter: embed_dim / preds_per_patch = %d channels; the CUDA head needs a multiple of 128, at most "
                "1024 (e.g. embed_dim=6144 with preds_per_patch=16)" % class_dim)
        if interpolate_mode != 'bilinear':
            raise NotImplementedError("ConvNeXtAdapter: interpolate_mode=%r; only 'bilinear' is implemented"
                                      % (interpolate_mode,))
        self.main_tasks = main_tasks
        self.patch_size = patch_size
        self.embed_dim = embed_dim
        self.preds_per_patch = preds_per_patch
        self.class_dim = class_dim
        self.num_classes = num_classes
        self.interpolate_mode = interpolate_mode
        self._side = s
        self._bound = None
        self._own_arena = False

        self.blocks = nn.Sequential(*[ConvNeXtBlock(dim=self.class_dim) for _ in range(depth)])
        self.final_layer = nn.Conv2d(self.class_dim, self.num_classes, 1)
        self.apply(self._init_weights)

    def init(self, dim_tokens_enc: int = 768):
        """Build proj_dec for encoder tokens of width dim_tokens_enc (called by MultiMAE.__init__)."""
        self.in_channels = dim_tokens_enc * len(self.main_tasks)
        self.proj_dec = nn.Linear(self.in_channels, self.embed_dim)
        self._init_weights(self.proj_dec)
        self._bound = None

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def bind(self, arena, prefix, on_grads_ready=None):
        self._own_arena = False
        self._bound = dict(arena=arena, prefix=prefix, on_grads_ready=on_grads_ready)

    def forward(self, encoder_tokens: torch.Tensor, input_info: Dict):
        assert hasattr(self, "proj_dec"), "Need to call init(dim_tokens_enc) function first"
        if not torch.is_tensor(encoder_tokens):
            raise NotImplementedError("multimae_b200: ConvNeXtAdapter takes the last layer's tokens "
                                      "(return_all_layers=False)")
        H, W = input_info['image_size']
        nh, nw = H // self.patch_size, W // self.patch_size
        for task in self.main_tasks:
            n_t = input_info['tasks'][task]['end_idx'] - input_info['tasks'][task]['start_idx']
            if n_t != nh * nw:
                raise ValueError("ConvNeXtAdapter: task %r has %d tokens, the %dx%d image has %d x %d = %d patches of %d"
                                 % (task, n_t, H, W, nh, nw, nh * nw, self.patch_size))
        if self._bound is None or self._bound["arena"].flat.device != encoder_tokens.device:
            # stand-alone use (outside MultiMAE / MultiViT): private gradient arena, zeroed on every training forward
            self.bind(Fn.GradArena([(n, p) for n, p in self.named_parameters() if p.requires_grad],
                                   encoder_tokens.device), "")
            self._own_arena = True
        params = [self.proj_dec.weight, self.proj_dec.bias, self.final_layer.weight, self.final_layer.bias]
        for blk in self.blocks:
            params += list(blk._params())
        save = torch.is_grad_enabled() and (encoder_tokens.requires_grad or any(p.requires_grad for p in params))
        if self._own_arena and save:
            self._bound["arena"].zero_()
        prefix = self._bound["prefix"]
        base = dict(self._bound, save=save, B=encoder_tokens.shape[0], nh=nh, nw=nw, s=self._side)
        starts = [input_info['tasks'][t]['start_idx'] for t in self.main_tasks]
        x = Fn.ConvNeXtProjFunction.apply(encoder_tokens, dict(base, n=nh * nw, starts=starts, channels=self.class_dim),
                                          self.proj_dec.weight, self.proj_dec.bias)
        for i, blk in enumerate(self.blocks):
            x = Fn.ConvNeXtBlockFunction.apply(x, dict(base, prefix="%sblocks.%d." % (prefix, i), eps=blk.norm.eps),
                                               *blk._params())
        return Fn.ConvNeXtTailFunction.apply(x, dict(base, num_classes=self.num_classes, H=H, W=W),
                                             self.final_layer.weight, self.final_layer.bias)


class SegmenterMaskTransformerAdapter(nn.Module):
    """Output adapter inspired by the Segmenter-Mask architecture (https://arxiv.org/abs/2105.05633): proj_dec of the main
    tasks' tokens, one learned token per class appended, `depth` transformer Blocks over the n + K tokens, decoder_norm, and
    the class map = LayerNorm over the classes of the cosine between every projected patch token and every projected class
    token, upsampled bilinearly to the image size.  Extra keyword arguments (stride_level, ...) are ignored, as by the
    reference.  Runs as SegmenterProjFunction -> functional.block_stack -> SegmenterTailFunction.

    The kernels need embed_dim to be a multiple of 128, at most 1024, with heads of 32 or 64 channels (768 with 12 heads in
    the reference's default), and 8 to 256 classes; anything else raises here."""

    def __init__(self, num_classes, depth: int = 2, num_heads: int = 12, embed_dim: int = 768, mlp_ratio=4,
                 drop_path_rate=0.1, drop_rate=0.0, attn_drop_rate=0.0, qkv_bias=True, main_tasks: Iterable[str] = ('rgb',),
                 patch_size: int = 16, norm_layer: nn.Module = partial(nn.LayerNorm, eps=1e-6), **kwargs):
        super().__init__()
        name = "SegmenterMaskTransformerAdapter"
        if embed_dim % 128 != 0 or embed_dim > 1024 or embed_dim % num_heads != 0 or embed_dim // num_heads not in (32, 64):
            raise NotImplementedError(
                "%s: embed_dim=%d with %d heads; the CUDA head needs embed_dim to be a multiple of 128, at most 1024, and "
                "heads of 32 or 64 channels (pass --decoder_dim 768 for the default 12 heads)" % (name, embed_dim, num_heads))
        if not 8 <= num_classes <= 256:
            raise NotImplementedError("%s: num_classes=%d; the mask kernel holds 8 to 256 classes" % (name, num_classes))
        self.main_tasks = main_tasks
        self.patch_size = patch_size
        self.embed_dim = embed_dim
        self.num_classes = num_classes
        self._bound = None
        self._own_arena = False

        self.cls_emb = nn.Parameter(torch.zeros(1, num_classes, embed_dim))
        trunc_normal_(self.cls_emb, std=0.02)

        self.patch_proj = nn.Linear(embed_dim, embed_dim, bias=False)
        self.classes_proj = nn.Linear(embed_dim, embed_dim, bias=False)

        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, drop=drop_rate,
                  attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer) for i in range(depth)])

        self.decoder_norm = norm_layer(embed_dim)
        self.mask_norm = norm_layer(num_classes)
        assert isinstance(self.decoder_norm, nn.LayerNorm), "multimae_b200: norm_layer must build nn.LayerNorm"
        self.apply(self._init_weights)

    def init(self, dim_tokens_enc: int = 768):
        """Build proj_dec for encoder tokens of width dim_tokens_enc (called by MultiMAE.__init__)."""
        self.in_channels = dim_tokens_enc * len(self.main_tasks)
        self.proj_dec = nn.Linear(self.in_channels, self.embed_dim)
        self._init_weights(self.proj_dec)
        self._bound = None

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def bind(self, arena, prefix, on_grads_ready=None):
        self._own_arena = False
        self._bound = dict(arena=arena, prefix=prefix, on_grads_ready=on_grads_ready)
        for i, blk in enumerate(self.blocks):
            blk.bind(arena, "%sblocks.%d." % (prefix, i), on_grads_ready)

    def forward(self, encoder_tokens: torch.Tensor, input_info: Dict):
        assert hasattr(self, "proj_dec"), "Need to call init(dim_tokens_enc) function first"
        if not torch.is_tensor(encoder_tokens):
            raise NotImplementedError("multimae_b200: SegmenterMaskTransformerAdapter takes the last layer's tokens "
                                      "(return_all_layers=False)")
        H, W = input_info['image_size']
        nh, nw = H // self.patch_size, W // self.patch_size
        for task in self.main_tasks:
            n_t = input_info['tasks'][task]['end_idx'] - input_info['tasks'][task]['start_idx']
            if n_t != nh * nw:
                raise ValueError("SegmenterMaskTransformerAdapter: task %r has %d tokens, the %dx%d image has %d x %d = %d "
                                 "patches of %d" % (task, n_t, H, W, nh, nw, nh * nw, self.patch_size))
        if self._bound is None or self._bound["arena"].flat.device != encoder_tokens.device:
            # stand-alone use (outside MultiMAE / MultiViT): private gradient arena, zeroed on every training forward
            self.bind(Fn.GradArena([(n, p) for n, p in self.named_parameters() if p.requires_grad],
                                   encoder_tokens.device), "")
            self._own_arena = True
        tail = [dict(self.named_parameters())[k] for k in Fn.SEGMENTER_TAIL_PARAM_NAMES]
        save = torch.is_grad_enabled() and (encoder_tokens.requires_grad or any(p.requires_grad for p in self.parameters()))
        if self._own_arena and save:
            self._bound["arena"].zero_()
        base = dict(self._bound, save=save, B=encoder_tokens.shape[0], nh=nh, nw=nw)
        starts = [input_info['tasks'][t]['start_idx'] for t in self.main_tasks]
        x = Fn.SegmenterProjFunction.apply(encoder_tokens, dict(base, n=nh * nw, starts=starts), self.proj_dec.weight,
                                           self.proj_dec.bias, self.cls_emb)
        x = Fn.block_stack(self.blocks, x)
        return Fn.SegmenterTailFunction.apply(x, dict(base, num_classes=self.num_classes, H=H, W=W,
                                                      eps_dec=self.decoder_norm.eps, eps_mask=self.mask_norm.eps), *tail)


class DPTOutputAdapter(nn.Module):
    """Placeholder so that the fine-tuning scripts import: the DPT head (multimae/output_adapters.py:576-) is not
    implemented on the CUDA path."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("multimae_b200: DPTOutputAdapter is not implemented; use --output_adapter convnext or "
                                  "segmenter")
