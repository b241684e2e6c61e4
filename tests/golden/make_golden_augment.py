"""Record augment.*.pt from the LIVE reference: DataAugmentationForMultiMAE (utils/datasets.py:66-111) on seeded synthetic
images (tests/augment_oracle.make_images: numpy -> PIL, no encoding, so only Pillow's resize decides the values).

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_augment.py

Input size 64, hflip 0.5, both mean / std choices.  Image sizes cover downscales of more than 2x, upscales from the
smallest crops, very thin images (get_params' centre-crop fallback: crops of a few pixels), and the identity size.  Per
case: the seed (random.seed and torch.manual_seed before the transform), the image size, the draws (flip, i, j, h, w) made
by the same calls the reference makes, and the reference's rgb / depth / semseg tensors."""
import os
import random
import sys
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from augment_oracle import make_images  # noqa: E402
from helpers import save_fixture  # noqa: E402

SIZES = [(375, 500), (500, 375), (480, 360), (300, 420), (256, 192), (40, 30), (24, 32), (17, 21), (64, 64), (64, 80),
         (3, 200), (200, 2), (20, 300), (400, 12), (1, 50), (90, 7)]


def main():
    import math
    import types
    sys.path.insert(0, os.environ["MULTIMAE_REFERENCE"])
    six = types.ModuleType("torch._six")        # utils/native_scaler.py imports a module removed in torch >= 2
    six.inf = math.inf
    sys.modules.setdefault("torch._six", six)
    import torchvision.transforms as transforms
    from utils.datasets import DataAugmentationForMultiMAE  # type: ignore
    cases = []
    for n in range(2 * len(SIZES)):
        h, w = SIZES[n % len(SIZES)]
        seed = 1000 + n
        default_norm = n % 2 == 1
        args = SimpleNamespace(imagenet_default_mean_and_std=default_norm, input_size=64, hflip=0.5)
        imgs = make_images(seed, h, w)
        random.seed(seed)
        torch.manual_seed(seed)
        flip = random.random() < args.hflip
        i, j, ch, cw = transforms.RandomResizedCrop.get_params(imgs["rgb"], scale=(0.2, 1.0), ratio=(0.75, 1.3333))
        random.seed(seed)
        torch.manual_seed(seed)
        out = DataAugmentationForMultiMAE(args)(dict(imgs))
        cases.append(dict(seed=seed, size=(h, w), default_norm=default_norm, draws=(bool(flip), i, j, ch, cw),
                          rgb=out["rgb"], depth=out["depth"], semseg=out["semseg"]))
    save_fixture(dict(input_size=64, hflip=0.5, cases=cases), os.path.join(HERE, "augment.pt"))


if __name__ == "__main__":
    main()
