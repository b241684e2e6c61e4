"""DataAugmentationForMultiMAE (EPFL-VILAB/MultiMAE utils/datasets.py:66-111) restated with PIL, numpy and torch only,
given its random draws (flip, i, j, h, w): the CPU oracle of the GPU augmentation (MMAE_GPU_AUGMENT).  It needs no
reference checkout and no torchvision; tests/golden/make_golden_augment.py checks it against the reference itself.

Also: the seeded synthetic images the fixtures and the tests are built from (numpy -> PIL, no encoding)."""
import numpy as np
import torch
from PIL import Image

DEFAULT_MEAN, DEFAULT_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
INCEPTION_MEAN, INCEPTION_STD = (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)


def make_images(seed, height, width, tasks=("rgb", "depth", "semseg"), num_classes=40):
    """{task: PIL image} of `height` x `width`: rgb 'RGB' (smooth gradients, noise and saturated blocks, so that bicubic
    overshoots clip), depth 'I;16' (the same structure over the full 16-bit range), semseg 'P' (blocky labels)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float64)
    out = {}
    for task in tasks:
        if task == "rgb":
            base = 127.5 + 100 * np.sin(xx[..., None] / (3 + 7 * rng.random(3)) + yy[..., None] / (5 + 9 * rng.random(3)))
            a = base + rng.normal(0, 25, (height, width, 3))
            a[rng.random((height, width)) < 0.05] = 255
            a[rng.random((height, width)) < 0.05] = 0
            out[task] = Image.fromarray(np.clip(np.rint(a), 0, 255).astype(np.uint8), "RGB")
        elif task == "depth":
            a = 32768 + 30000 * np.cos(xx / (4 + 6 * rng.random()) - yy / (3 + 5 * rng.random()))
            a = a + rng.normal(0, 2500, (height, width))
            a[rng.random((height, width)) < 0.05] = 65535
            a[rng.random((height, width)) < 0.05] = 0
            a = np.clip(np.rint(a), 0, 65535).astype(np.uint16)
            out[task] = Image.frombuffer("I;16", (width, height), a.astype("<u2").tobytes(), "raw", "I;16", 0, 1)
        else:
            cells = rng.integers(0, num_classes, (height // 7 + 1, width // 5 + 1)).astype(np.uint8)
            a = np.ascontiguousarray(cells.repeat(7, 0).repeat(5, 1)[:height, :width])
            out[task] = Image.frombytes("P", (width, height), a.tobytes())
    return out


def augment(task_dict, draws, input_size, mean=INCEPTION_MEAN, std=INCEPTION_STD):
    """The reference transform of one sample for the draws (flip, i, j, h, w): crop, resize to input_size (Pillow's
    default filter for the mode), flip, then to tensors: rgb normalised fp32 [3,S,S], depth fp32 [1,S,S] (/ 2**16),
    semseg int64 [S/4,S/4] (a second nearest resize)."""
    flip, i, j, h, w = draws
    imgs = {}
    for task, img in task_dict.items():
        img = img.crop((j, i, j + w, i + h)).resize((input_size, input_size))
        if flip:
            img = img.transpose(Image.Transpose.FLIP_LEFT_RIGHT)
        imgs[task] = img
    out = {}
    for task, img in imgs.items():
        if task == "depth":
            out[task] = torch.Tensor(np.array(img) / 2 ** 16).unsqueeze(0)
        elif task == "rgb":
            t = torch.from_numpy(np.array(img)).permute(2, 0, 1).contiguous().to(torch.float32).div(255)
            out[task] = t.sub_(torch.as_tensor(mean, dtype=torch.float32)[:, None, None]).div_(
                torch.as_tensor(std, dtype=torch.float32)[:, None, None])
        else:
            s4 = int(input_size * 0.25)
            out[task] = torch.from_numpy(np.array(img.resize((s4, s4)))).to(torch.long)
    return out
