"""Record cls_augment.*.pt from the LIVE reference: utils/datasets.py:build_transform (train: RandomResizedCropAndInterpolation,
RandomHorizontalFlip, RandAugment, ToTensor, Normalize; eval: Resize + CenterCrop, ToTensor, Normalize) on seeded synthetic
images (tests/cls_augment_oracle.make_image: numpy -> PIL, no encoding).

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_cls_augment.py

Input size 48.  Per case: the transform's arguments, the image size, the seed (random.seed, np.random.seed and
torch.manual_seed before the transform), the reference's tensor and a digest of the three RNG states after it (Python's
random, NumPy's global RandomState, torch's CPU generator)."""
import hashlib
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from cls_augment_oracle import make_image  # noqa: E402
from helpers import save_fixture  # noqa: E402

SIZES = [(375, 500), (500, 375), (120, 90), (64, 64), (37, 53), (300, 40), (20, 300), (70, 71)]
CONFIGS = [  # (aa, train_interpolation, imagenet_default_mean_and_std)
    ("rand-m9-mstd0.5-inc1", "bicubic", True),
    ("rand-m9-mstd0.5-inc1", "bicubic", False),
    ("rand-m9-mstd0.5-inc1", "bilinear", True),
    ("rand-m9-mstd0.5-inc1", "random", True),
    ("rand-m10-n3-mstd0.5", "bicubic", True),
    ("rand-m7-n1", "random", False),
    ("rand-m9-mstd0.5-inc1-w0", "bicubic", True),
    ("rand-m15-mmax30-mstd3-n2-inc1", "random", True),
    ("rand-m25-mmax30-n3-inc1", "bilinear", False),      # magnitudes above 10: LUT op arguments out of their range
    ("rand-m25-mmax30-n3", "random", True),
]


def rng_digest():
    """sha256 of the three generators' states (Python's random, NumPy's global RandomState, torch's default CPU)."""
    h = hashlib.sha256(repr(random.getstate()).encode())
    st = np.random.get_state()
    h.update(st[1].tobytes() + repr(st[2:]).encode())
    h.update(torch.get_rng_state().numpy().tobytes())
    return h.hexdigest()


def main():
    import math
    import types
    sys.path.insert(0, os.environ["MULTIMAE_REFERENCE"])
    six = types.ModuleType("torch._six")        # utils/native_scaler.py imports a module removed in torch >= 2
    six.inf = math.inf
    sys.modules.setdefault("torch._six", six)
    from PIL import Image
    from utils.datasets import build_transform  # type: ignore
    cases = []
    n = 0
    for aa, interp, default_norm in CONFIGS:
        for rep in range(6):
            h, w = SIZES[(n + rep) % len(SIZES)]
            args = SimpleNamespace(input_size=48, imagenet_default_mean_and_std=default_norm, color_jitter=0.4, aa=aa,
                                   train_interpolation=interp, reprob=0.0, remode="pixel", recount=1, crop_pct=None)
            t = build_transform(True, args)
            seed = 5000 + n
            img = Image.fromarray(make_image(seed, h, w))
            random.seed(seed)
            np.random.seed(seed)
            torch.manual_seed(seed)
            out = t(img)
            cases.append(dict(train=True, aa=aa, interp=interp, default_norm=default_norm, size=(h, w), seed=seed,
                              out=out, rng=rng_digest()))
            n += 1
    for k, (h, w) in enumerate(SIZES):
        args = SimpleNamespace(input_size=48, imagenet_default_mean_and_std=k % 2 == 0, crop_pct=None)
        seed = 9000 + k
        out = build_transform(False, args)(Image.fromarray(make_image(seed, h, w)))
        cases.append(dict(train=False, default_norm=k % 2 == 0, size=(h, w), seed=seed, out=out))
    save_fixture(dict(input_size=48, cases=cases), os.path.join(HERE, "cls_augment.pt"))


if __name__ == "__main__":
    main()
