"""Counterpart of the reference's ``tools/`` for the hot path: optimizer / scheduler / training-mode builders
(tools/utils.py), the train / test loops (tools/scripts.py, tools/interactive_segmentation_scripts.py) and the
``--work-dir`` entry points train_classification_model, train_imagenet21k_classification_model,
train_distill_classification_model, train_mae_self_supervised_model, train_interactive_segmentation_distill_encoder_model
and test_classification_model, whose shared loop is tools/driver.py."""
