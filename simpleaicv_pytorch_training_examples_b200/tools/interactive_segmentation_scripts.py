"""Step bodies of the interactive-segmentation training loops that only need the SAM image encoder
(tools/interactive_segmentation_scripts.py:21-199 train_distill_sam_encoder).  train_sam_segmentation (:274-564) needs
the prompt encoder / mask decoder and SAMLoss, which are not on the H100 path yet (SURVEY.md 8 f1)."""
from ..classification.common import AverageMeter  # noqa: F401  (re-exported like the reference module)
from .scripts import train_epoch_with_loss_terms
from .utils import unwrap


def train_distill_sam_encoder(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config):
    """One epoch of encoder distillation: `model(images)` returns (teacher_outputs, student_outputs), the criterion a
    dict of loss terms (reference :21-199; same guards, accumulation, clipping and per-iteration LR as train_detection)."""
    model.train()
    if getattr(config, 'freeze_teacher', False):
        unwrap(model).teacher.eval()

    def compute(data):
        images = data['image']
        tea_outputs, stu_outputs = model(images)
        return criterion(tea_outputs, stu_outputs), (images,), images.size(0)

    return train_epoch_with_loss_terms(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute,
                                       total_name='loss')


def train_sam_segmentation(*args, **kwargs):
    raise NotImplementedError('train_sam_segmentation needs the SAM prompt encoder / mask decoder and SAMLoss, which are not '
                              'built on the H100 path yet (SURVEY.md 8 f1)')
