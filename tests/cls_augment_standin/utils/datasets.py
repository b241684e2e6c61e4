"""utils/datasets.py of the reference, as far as classification data goes (see __init__.py)."""
from torchvision import datasets

import cls_augment_oracle
from multimae_b200 import data as D


class _CpuTransform:
    def __init__(self, draws, is_train):
        self.draws, self.is_train = draws, is_train
        self.transforms = [self]

    def __call__(self, img):
        t, S = self.draws, self.draws.input_size
        if self.is_train:
            return cls_augment_oracle.pil_train_sample(t(img), S, t.mean, t.std, t.fill)
        return cls_augment_oracle.pil_eval_sample(img, t.resize, S, t.mean, t.std)


def build_transform(is_train, args):
    if is_train:
        return _CpuTransform(D.ClsTrainTransform(args), True)
    if args.crop_pct is None:
        args.crop_pct = 224 / 256 if args.input_size < 384 else 1.0
    return _CpuTransform(D.ClsEvalTransform(args), False)


def build_dataset(is_train, args):
    transform = build_transform(is_train, args)
    for t in transform.transforms:
        print(t)
    root = args.data_path if is_train else args.eval_data_path
    return datasets.ImageFolder(root, transform=transform), args.nb_classes
