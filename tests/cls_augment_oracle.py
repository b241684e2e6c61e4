"""The C-side arithmetic of the classification fine-tuning transform (utils/transforms_factory.py:
RandomResizedCropAndInterpolation, RandomHorizontalFlip, RandAugment, ToTensor, Normalize) restated in numpy on uint8
[H, W, 3] images, given the op records multimae_b200.data makes in the workers: the CPU oracle of the GPU path
(MMAE_GPU_AUGMENT, mmae_cls_augment_batch).  Pillow's Python code is restated in data.py; what is restated here is what
Pillow does in C (resampling, LUTs, ImagingBlend, the 3x3 filter, the affine transform filters), and
tests/test_cls_augment_host.py proves it bitwise against the installed Pillow.  Test infrastructure only."""
import numpy as np
import torch

from multimae_b200 import data as D

F32 = np.float32


def resize(crop, size, filt):
    """Pillow's Image.resize of a uint8 [h, w, 3] crop to size x size with `filt` (D.FILTER_BILINEAR / D.FILTER_BICUBIC):
    horizontal pass with 22-bit fixed-point weights, clip, then the vertical pass."""
    h, w = crop.shape[:2]
    return _pass(_pass(crop.astype(np.int64), _table(filt, w, size), 1), _table(filt, h, size), 0).astype(np.uint8)


def _table(filt, n_in, n_out):
    bounds, w = D.resample_coeffs(filt, n_in, n_out)
    return bounds, D.fixed_point_coeffs(w)


def resize_sliced(img, rows, cols):
    """The eval path: resample `img` through the (bounds, fixed-point weights) row and column tables."""
    return _pass(_pass(img.astype(np.int64), cols, 1), rows, 0).astype(np.uint8)


def _pass(a, table, axis):
    bounds, fixed = table
    out = []
    for k in range(len(bounds)):
        lo, cnt = int(bounds[k, 0]), int(bounds[k, 1])
        src = a[:, lo:lo + cnt] if axis == 1 else a[lo:lo + cnt]
        wk = fixed[k, :cnt].astype(np.int64)
        s = (src * (wk[None, :, None] if axis == 1 else wk[:, None, None])).sum(axis) + (1 << 21)
        out.append(np.clip(s >> 22, 0, 255))
    return np.stack(out, axis)


def hflip(img):
    return np.ascontiguousarray(img[:, ::-1])


def lut(img, table):
    """ImageOps / Image.point with a 256-entry table per channel: table [3, 256] or [256]."""
    t = np.asarray(table)
    if t.ndim == 1:
        return t.astype(np.uint8)[img]
    return np.stack([t[c].astype(np.uint8)[img[..., c]] for c in range(3)], -1)


def luma(img):
    """Pillow's RGB -> L: (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16."""
    i = img.astype(np.int64)
    return ((i[..., 0] * 19595 + i[..., 1] * 38470 + i[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def histograms(img):
    return [np.bincount(img[..., c].reshape(-1), minlength=256) for c in range(3)]


def blend(degenerate, img, alpha):
    """ImagingBlend(degenerate, img, (float) alpha): in1 + alpha * (in2 - in1) in float32, truncated, clipped outside
    [0, 1]."""
    a = F32(alpha)
    in1 = degenerate.astype(np.int32)
    t = in1.astype(F32) + a * (img.astype(np.int32) - in1).astype(F32)
    if 0.0 <= a <= 1.0:
        return t.astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.clip(t, 0, 255).astype(np.uint8))).astype(np.uint8)


def smooth(img):
    """ImageFilter.SMOOTH (3x3, (1,1,1,1,5,1,1,1,1) / 13 in float32, offset 0.5 added once, truncated and clipped);
    border pixels are copied."""
    k = np.array([1, 1, 1, 1, 5, 1, 1, 1, 1], F32) / F32(13)
    a = img.astype(F32)
    out = img.copy()
    H, W = img.shape[:2]
    if H < 3 or W < 3:
        return out

    def k3(row, kk):            # KERNEL1x3 on rows of a: (in[x-1] * k0 + in[x] * k1) + in[x+1] * k2
        return (row[:, :-2] * kk[0] + row[:, 1:-1] * kk[1]) + row[:, 2:] * kk[2]
    ss = np.full((H - 2, W - 2, 3), F32(0.5), F32)
    ss = ss + k3(a[2:], k[0:3])
    ss = ss + k3(a[1:-1], k[3:6])
    ss = ss + k3(a[:-2], k[6:9])
    v = np.where(ss <= 0, 0, np.where(ss >= 255, 255, np.clip(ss, 0, 255).astype(np.uint8)))
    out[1:-1, 1:-1] = v
    return out


def affine(img, m, filt, fill):
    """Image.transform(size, AFFINE, m, filt, fillcolor=fill): ImagingGenericTransform with affine_transform and the
    bilinear / bicubic 32RGB filters; pixels whose source falls outside the image keep the fill colour."""
    H, W = img.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    xs, ys = xs + 0.5, ys + 0.5
    xin = (m[0] * xs + m[1] * ys) + m[2]
    yin = (m[3] * xs + m[4] * ys) + m[5]
    inside = (xin >= 0.0) & (xin < W) & (yin >= 0.0) & (yin < H)
    xin, yin = xin - 0.5, yin - 0.5
    x = np.floor(xin).astype(np.int64)
    y = np.floor(yin).astype(np.int64)
    dx, dy = xin - x, yin - y
    a = img.astype(np.int64)
    out = np.empty_like(img)
    for c in range(3):
        ch = a[..., c]

        def at(yy, xx):
            return ch[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        if filt == D.FILTER_BILINEAR:
            def row(yy):
                p0, p1 = at(yy, x), at(yy, x + 1)
                return p0 + (p1 - p0) * dx
            v1 = row(y)
            ok = (y + 1 >= 0) & (y + 1 < H)
            v2 = row(y + 1)
            v = np.where(ok, v1 + (v2 - v1) * dy, v1)
            out[..., c] = v.astype(np.uint8)
        else:
            xb, yb = x - 1, y - 1

            def cub(v1, v2, v3, v4, d):
                p1 = v2
                p2 = -v1 + v3
                p3 = 2 * (v1 - v2) + v3 - v4
                p4 = -v1 + v2 - v3 + v4
                return p1 + d * (p2 + d * (p3 + d * p4))

            def row(yy):
                return cub(at(yy, xb), at(yy, xb + 1), at(yy, xb + 2), at(yy, xb + 3), dx)
            r1 = row(yb)
            r2 = np.where((yb + 1 >= 0) & (yb + 1 < H), row(yb + 1), r1)
            r3 = np.where((yb + 2 >= 0) & (yb + 2 < H), row(yb + 2), r2)
            r4 = np.where((yb + 3 >= 0) & (yb + 3 < H), row(yb + 3), r3)
            v = cub(r1, r2, r3, r4, dy)
            out[..., c] = np.where(v <= 0, 0, np.where(v >= 255, 255, np.clip(v, 0, 255).astype(np.uint8)))
        out[..., c] = np.where(inside, out[..., c], fill[c])
    return out


def apply_op(img, op, fill):
    """One RandAugment op record (D.ClsOp) on a uint8 [S, S, 3] image."""
    k = op.kind
    if k == D.OP_IDENTITY:
        return img.copy()
    if k == D.OP_INVERT:
        return lut(img, 255 - np.arange(256))
    if k == D.OP_POSTERIZE:
        return lut(img, np.arange(256) & ~(2 ** (8 - op.iarg) - 1))
    if k == D.OP_SOLARIZE:
        i = np.arange(256)
        return lut(img, np.where(i < op.iarg, i, 255 - i))
    if k == D.OP_SOLARIZE_ADD:
        i = np.arange(256)
        return lut(img, np.where(i < 128, np.minimum(255, i + op.iarg), i))
    if k == D.OP_AUTOCONTRAST:
        return lut(img, [D.autocontrast_lut(h) for h in histograms(img)])
    if k == D.OP_EQUALIZE:
        return lut(img, [D.equalize_lut(h) for h in histograms(img)])
    if k == D.OP_COLOR:
        g = luma(img)
        return blend(np.stack([g, g, g], -1), img, op.factor)
    if k == D.OP_CONTRAST:
        mean = D.contrast_mean(np.bincount(luma(img).reshape(-1), minlength=256))
        return blend(np.full_like(img, mean), img, op.factor)
    if k == D.OP_BRIGHTNESS:
        return blend(np.zeros_like(img), img, op.factor)
    if k == D.OP_SHARPNESS:
        return blend(smooth(img), img, op.factor)
    if k == D.OP_AFFINE:
        return affine(img, op.matrix, op.filter, fill)
    if k == D.OP_TRANSPOSE:
        if op.iarg == 180:
            return np.ascontiguousarray(img[::-1, ::-1])
        if op.iarg == 90:                         # Transpose.ROTATE_90 (counter-clockwise)
            return np.ascontiguousarray(np.rot90(img, 1))
        return np.ascontiguousarray(np.rot90(img, 3))
    raise ValueError(k)


def to_tensor_normalize(img, mean, std):
    t = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).contiguous().to(torch.float32).div(255)
    return t.sub_(torch.as_tensor(mean, dtype=torch.float32)[:, None, None]).div_(
        torch.as_tensor(std, dtype=torch.float32)[:, None, None])


def train_sample(rec, size, mean, std, fill):
    """The whole training transform of one worker record (D.ClsSample): resize, flip, ops, normalise."""
    img = resize(rec.crop, size, rec.filter)
    if rec.flip:
        img = hflip(img)
    for op in rec.ops:
        img = apply_op(img, op, fill)
    return to_tensor_normalize(img, mean, std)


def eval_sample(rec, size, mean, std):
    rows = D.sliced_table(D.FILTER_BICUBIC, *rec.rows, size)[:2]
    cols = D.sliced_table(D.FILTER_BICUBIC, *rec.cols, size)[:2]
    return to_tensor_normalize(resize_sliced(rec.crop, rows, cols), mean, std)


def make_image(seed, height, width, flat=None):
    """A seeded uint8 RGB image: gradients, noise and saturated dots (or one flat colour `flat`)."""
    if flat is not None:
        return np.broadcast_to(np.asarray(flat, np.uint8), (height, width, 3)).copy()
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    base = 127.5 + 100 * np.sin(xx[..., None] / (3 + 7 * rng.random(3)) + yy[..., None] / (5 + 9 * rng.random(3)))
    a = base + rng.normal(0, 25, (height, width, 3))
    a[rng.random((height, width)) < 0.05] = 255
    a[rng.random((height, width)) < 0.05] = 0
    return np.clip(np.rint(a), 0, 255).astype(np.uint8)



def pil_op(img, op, fill):
    """The same op record applied with the Pillow calls the reference makes (a PIL image in and out)."""
    from PIL import Image, ImageEnhance, ImageOps
    k = op.kind
    if k == D.OP_IDENTITY:
        return img
    if k == D.OP_INVERT:
        return ImageOps.invert(img)
    if k == D.OP_POSTERIZE:
        return ImageOps.posterize(img, op.iarg)
    if k == D.OP_SOLARIZE:
        return ImageOps.solarize(img, op.iarg)
    if k == D.OP_SOLARIZE_ADD:
        return img.point([min(255, i + op.iarg) if i < 128 else i for i in range(256)] * 3)
    if k == D.OP_AUTOCONTRAST:
        return ImageOps.autocontrast(img)
    if k == D.OP_EQUALIZE:
        return ImageOps.equalize(img)
    if k in (D.OP_COLOR, D.OP_CONTRAST, D.OP_BRIGHTNESS, D.OP_SHARPNESS):
        cls = {D.OP_COLOR: ImageEnhance.Color, D.OP_CONTRAST: ImageEnhance.Contrast,
               D.OP_BRIGHTNESS: ImageEnhance.Brightness, D.OP_SHARPNESS: ImageEnhance.Sharpness}[k]
        return cls(img).enhance(op.factor)
    if k == D.OP_AFFINE:
        return img.transform(img.size, Image.AFFINE, op.matrix, resample=op.filter, fillcolor=fill)
    return img.transpose({90: Image.Transpose.ROTATE_90, 180: Image.Transpose.ROTATE_180,
                          270: Image.Transpose.ROTATE_270}[op.iarg])


def pil_train_sample(rec, size, mean, std, fill):
    """train_sample with Pillow doing the pixel work, as the reference's transform does."""
    from PIL import Image
    img = Image.fromarray(rec.crop).resize((size, size), rec.filter)
    if rec.flip:
        img = img.transpose(Image.Transpose.FLIP_LEFT_RIGHT)
    for op in rec.ops:
        img = pil_op(img, op, fill)
    return to_tensor_normalize(np.asarray(img), mean, std)


def pil_eval_sample(img, resize, size, mean, std):
    """Resize(resize, bicubic) + CenterCrop(size) of a PIL image with Pillow, then to_tensor / normalize."""
    from PIL import Image
    W, H = img.size
    short, long = (W, H) if W <= H else (H, W)
    new_long = int(resize * long / short)
    new_w, new_h = (resize, new_long) if W <= H else (new_long, resize)
    img = img.resize((new_w, new_h), Image.BICUBIC)
    top, left = int(round((new_h - size) / 2.0)), int(round((new_w - size) / 2.0))
    return to_tensor_normalize(np.asarray(img.crop((left, top, left + size, top + size))), mean, std)
