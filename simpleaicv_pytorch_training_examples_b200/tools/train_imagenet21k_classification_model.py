"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_imagenet21k_classification_model --work-dir DIR``

Drop-in for the reference's tools/train_imagenet21k_classification_model.py (the three configs under
00.classification_training/imagenet21k/): the loop of train_classification_model with the semantic-softmax epoch bodies.
``<work-dir>/train_config.py`` keeps the reference's ImageNet21KSemanticTreeLabelDataset; its ``backbones`` / ``losses``
imports point at this package, whose SemanticSoftmaxLoss runs on the semantic tree's device tables.
"""
from .scripts import test_imagenet21k_classification, train_imagenet21k_classification
from .train_classification_model import main as _main


def main():
    _main(train_imagenet21k_classification, test_imagenet21k_classification)


if __name__ == '__main__':
    main()
