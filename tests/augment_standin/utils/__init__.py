"""Stand-in for the part of the reference's `utils` package (EPFL-VILAB/MultiMAE, utils/) that run_pretraining_multimae.py
uses to build its data: utils.datasets.build_multimae_pretraining_dataset with DataAugmentationForMultiMAE and
MultiTaskImageFolder, restated so that the tests run without a reference checkout.  The transform is
tests/augment_oracle.py after the reference's draws (random.random() < hflip, then RandomResizedCrop.get_params, here
multimae_b200.data.random_resized_crop_params, which the golden fixtures hold to torchvision's).

Only the tests import it, with this directory put on sys.path; nothing else here is named `utils`."""
from . import datasets  # noqa: F401
