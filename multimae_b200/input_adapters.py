"""Input adapters with the reference's constructor / attribute / state_dict contract (multimae/input_adapters.py).

Inside `MultiMAE.forward` the adapters are not called one by one: the model embeds only the visible patches of all
modalities with one K-concatenated wgmma GEMM (functional.EmbedFunction).  Calling an adapter directly embeds all of
its patches through the same kernels (MultiViT / stand-alone use)."""
from typing import Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from .multimae_utils import build_2d_sincos_posemb, pair, trunc_normal_


class _PosEmbCache:
    """Resized positional table rows [nh*nw, D] for the frozen sin-cos parameter (reference re-runs F.interpolate every
    forward: multimae/input_adapters.py:113,235; the table is constant, so it is computed once per size/device).

    A trainable table of an input adapter never comes here: the embedding resizes it on the device every call and returns
    its gradient (functional.EmbedFunction).  The output adapters have no such path and refuse one."""

    def _resized_pos(self, nh, nw, mode):
        if self.pos_emb.requires_grad:
            raise NotImplementedError("multimae_b200: learnable_pos_emb=True is outside the pre-training hot path")
        key = (nh, nw, mode, self.pos_emb.device, self.pos_emb._version, self.pos_emb.data_ptr())
        cache = self.__dict__.setdefault("_pos_cache", {})
        if key not in cache:
            cache.clear()
            with torch.no_grad():
                kw = dict(align_corners=False) if mode == "bicubic" else {}
                t = F.interpolate(self.pos_emb.detach().float(), size=(nh, nw), mode=mode, **kw)
                cache[key] = t.flatten(2).transpose(1, 2)[0].contiguous()
        return cache[key]


class _PatchTokenAdapter(nn.Module, _PosEmbCache):
    """What both input adapters share: the patch geometry derived from (stride_level, patch_size_full), the frozen or
    learnable position table built at `init(dim_tokens)` time, and the entry into the gather-first embedding kernels.
    Attribute names (`stride_level`, `P_H`, `P_W`, `image_size`, `dim_tokens`, `pos_emb`, `proj`) are the ones
    MultiMAE.forward, the converters and checkpoints of the reference read (multimae/input_adapters.py:41-95, 141-213)."""

    is_semseg = False
    pos_mode = "bicubic"           # how the table is resized to another grid (:113 bicubic, :235 bilinear)

    def _set_geometry(self, stride_level, patch_size_full, dim_tokens, sincos_pos_emb, learnable_pos_emb, image_size):
        self.stride_level = stride_level
        self.patch_size_full = pair(patch_size_full)
        self.dim_tokens = dim_tokens
        self.sincos_pos_emb = sincos_pos_emb
        self.learnable_pos_emb = learnable_pos_emb
        self.image_size = pair(image_size)
        self.P_H, self.P_W = (max(1, side // stride_level) for side in self.patch_size_full)

    def _make_pos_emb(self):
        """[1, D, h, w] table over the adapter's own image_size grid, registered under the reference's name."""
        grid_h = self.image_size[0] // (self.stride_level * self.P_H)
        grid_w = self.image_size[1] // (self.stride_level * self.P_W)
        if self.sincos_pos_emb:
            self.pos_emb = nn.Parameter(build_2d_sincos_posemb(h=grid_h, w=grid_w, embed_dim=self.dim_tokens),
                                        requires_grad=self.learnable_pos_emb)
        else:
            self.pos_emb = nn.Parameter(torch.zeros(1, self.dim_tokens, grid_h, grid_w))
            trunc_normal_(self.pos_emb, std=0.02)

    def _make_proj(self, in_channels):
        # non-overlapping P x P convolution == one linear map per patch; the kernels read its weight as [D, C*P*P]
        self.proj = nn.Conv2d(in_channels=in_channels, out_channels=self.dim_tokens, kernel_size=(self.P_H, self.P_W),
                              stride=(self.P_H, self.P_W))

    def grid(self, x):
        """Patch grid (nh, nw) of an input [..., H, W] (the reference's divisibility asserts, :105-106 / :223-225)."""
        H, W = x.shape[-2:]
        assert self.dim_tokens is not None, "Need to call init(dim_tokens) function first"
        assert (H % self.P_H == 0) and (W % self.P_W == 0), \
            f"Image sizes {H}x{W} must be divisible by patch sizes {self.P_H}x{self.P_W}"
        return H // self.P_H, W // self.P_W

    def forward(self, x):
        from .multimae import embed_all_patches
        return embed_all_patches(self, x)


class PatchedInputAdapter(_PatchTokenAdapter):
    """Adapter for spatial inputs: patchify (Conv2d k=s=P == per-patch linear) + 2D sin-cos pos-emb.
    Reference: multimae/input_adapters.py:27-119."""

    def __init__(self, num_channels: int, stride_level: int, patch_size_full: Union[int, Tuple[int, int]],
                 dim_tokens: Optional[int] = None, sincos_pos_emb: bool = True, learnable_pos_emb: bool = False,
                 image_size: Union[int, Tuple[int]] = 224):
        super().__init__()
        self.num_channels = num_channels
        self._set_geometry(stride_level, patch_size_full, dim_tokens, sincos_pos_emb, learnable_pos_emb, image_size)
        self.num_patches = (self.image_size[0] // patch_size_full) * (self.image_size[1] // patch_size_full)
        if dim_tokens is not None:
            self.init(dim_tokens=dim_tokens)

    def init(self, dim_tokens: int = 768):
        self.dim_tokens = dim_tokens
        self._make_pos_emb()
        self._make_proj(self.num_channels)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_emb"}

    def embed_channels(self):
        return self.num_channels


class SemSegInputAdapter(_PatchTokenAdapter):
    """Adapter for semantic-segmentation maps: class-embedding lookup + patchify + pos-emb.
    Reference: multimae/input_adapters.py:122-241."""

    is_semseg = True
    pos_mode = "bilinear"

    def __init__(self, num_classes: int, stride_level: int, patch_size_full: Union[int, Tuple[int, int]],
                 dim_tokens: Optional[int] = None, sincos_pos_emb: int = True, learnable_pos_emb: int = False,
                 image_size: Union[int, Tuple[int]] = 224, dim_class_emb: int = 64, interpolate_class_emb: bool = False,
                 emb_padding_idx: int = None):
        super().__init__()
        if interpolate_class_emb:
            raise NotImplementedError("multimae_b200: interpolate_class_emb=True is outside the pre-training hot path")
        self.num_classes = num_classes + (1 if emb_padding_idx is not None else 0)     # the padding class gets a row too
        self.dim_class_emb = dim_class_emb
        self.interpolate_class_emb = interpolate_class_emb
        self.emb_padding_idx = emb_padding_idx
        self._set_geometry(stride_level, patch_size_full, dim_tokens, sincos_pos_emb, learnable_pos_emb, image_size)
        if dim_tokens is not None:
            self.init(dim_tokens=dim_tokens)

    def init(self, dim_tokens: int = 768):
        self.dim_tokens = dim_tokens
        self._make_pos_emb()
        self.class_emb = nn.Embedding(num_embeddings=self.num_classes, embedding_dim=self.dim_class_emb,
                                      padding_idx=self.emb_padding_idx)
        trunc_normal_(self.class_emb.weight, std=0.02)
        self._make_proj(self.dim_class_emb)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {"pos_emb", "class_emb"}

    def embed_channels(self):
        return self.dim_class_emb
