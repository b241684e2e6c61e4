"""utils/datasets.py + utils/dataset_folder.py of the reference, as far as pre-training data goes (see __init__.py)."""
import os
import random

from PIL import Image

import augment_oracle
from multimae_b200.data import random_resized_crop_params


class DataAugmentationForMultiMAE:
    def __init__(self, args):
        default = args.imagenet_default_mean_and_std
        self.mean = augment_oracle.DEFAULT_MEAN if default else augment_oracle.INCEPTION_MEAN
        self.std = augment_oracle.DEFAULT_STD if default else augment_oracle.INCEPTION_STD
        self.input_size, self.hflip = args.input_size, args.hflip

    def __call__(self, task_dict):
        flip = random.random() < self.hflip
        first = next(iter(task_dict.values()))
        i, j, h, w = random_resized_crop_params(first.height, first.width)
        return augment_oracle.augment(task_dict, (flip, i, j, h, w), self.input_size, self.mean, self.std)


class MultiTaskImageFolder:
    """root/<task>/<class>/<file>, the same file names under every task; targets are class indices in sorted order."""

    def __init__(self, root, tasks, transform=None):
        self.root, self.tasks, self.transform = root, list(tasks), transform
        classes = sorted(d.name for d in os.scandir(os.path.join(root, self.tasks[0])) if d.is_dir())
        self.samples = {t: [] for t in self.tasks}
        for ci, c in enumerate(classes):
            for name in sorted(os.listdir(os.path.join(root, self.tasks[0], c))):
                stem = os.path.splitext(name)[0]
                for t in self.tasks:
                    match = [f for f in os.listdir(os.path.join(root, t, c)) if os.path.splitext(f)[0] == stem]
                    self.samples[t].append((os.path.join(root, t, c, match[0]), ci))

    def __len__(self):
        return len(self.samples[self.tasks[0]])

    def __getitem__(self, index):
        sample = {}
        for t in self.tasks:
            path, target = self.samples[t][index]
            img = Image.open(path)
            img = img.convert("RGB") if t == "rgb" else img
            sample[t] = img.convert("P") if "semseg" in t else img
        if self.transform is not None:
            sample = self.transform(sample)
        return sample, target


def build_multimae_pretraining_dataset(args):
    return MultiTaskImageFolder(args.data_path, args.all_domains, transform=DataAugmentationForMultiMAE(args))
