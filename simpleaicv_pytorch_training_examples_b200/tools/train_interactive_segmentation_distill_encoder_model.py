"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_interactive_segmentation_distill_encoder_model --work-dir DIR``

Drop-in for the reference's tools/train_interactive_segmentation_distill_encoder_model.py (13.0.encoder_distill_training):
``config.model`` is an ``interactive_segmentation.distill_model`` encoder-distillation model and ``config.train_criterion``
its ``distill_losses.MSELoss``.  There is no test set: the student is saved every ``config.save_interval`` epochs as
``student_model_epoch_{epoch}.pth`` and as ``best_student.pth`` at the lowest epoch train loss.  No EMA model, as in the
reference.
"""
import os

import torch

from .driver import Task, rename_if_exists, run
from .interactive_segmentation_scripts import train_distill_sam_encoder
from .utils import unwrap


class DistillEncoderTask(Task):
    keep_ema = False

    def __init__(self):
        super().__init__(train_distill_sam_encoder)
        self.state = {'best_loss': 1e9, 'train_loss': 0.}

    def resume_info(self):
        return f'best_loss {self.state["best_loss"]:.4f}'

    def end_epoch(self, epoch, train_loss, result, model, eval_model, checkpoint_dir, config):
        student = unwrap(model).student
        if epoch % config.save_interval == 0:
            torch.save(student.state_dict(), os.path.join(checkpoint_dir, f'student_model_epoch_{epoch}.pth'))
        self.state['train_loss'] = train_loss
        if train_loss < self.state['best_loss']:
            self.state['best_loss'] = train_loss
            torch.save(student.state_dict(), os.path.join(checkpoint_dir, 'best_student.pth'))
        return f'best_loss {self.state["best_loss"]:.4f}, '

    def finish(self, checkpoint_dir, config):
        rename_if_exists(checkpoint_dir, 'best_student.pth',
                         f'student-epoch{config.epochs}-loss{self.state["best_loss"]:.3f}.pth')


def main():
    run(DistillEncoderTask(), 'H100 interactive segmentation encoder distillation training')


if __name__ == '__main__':
    main()
