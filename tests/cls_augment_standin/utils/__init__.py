"""Stand-in for the part of the reference's `utils` package (EPFL-VILAB/MultiMAE, utils/) that run_finetuning_cls.py
uses to build its data: utils.datasets.build_dataset and build_transform, restated so that the tests run without a
reference checkout.  The transform is the workers' draws (multimae_b200.data.ClsTrainTransform / ClsEvalTransform, which
the golden fixtures hold to the reference's) followed by the same Pillow calls as the reference's
(tests/cls_augment_oracle.py: pil_train_sample, pil_eval_sample).

Only the tests import it, with this directory put on sys.path; nothing else here is named `utils`."""
from . import datasets  # noqa: F401
