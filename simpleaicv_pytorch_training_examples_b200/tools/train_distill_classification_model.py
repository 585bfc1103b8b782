"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_distill_classification_model --work-dir DIR``

Drop-in for the reference's tools/train_distill_classification_model.py (the four configs under
01.distillation_training/imagenet/): ``config.model`` is a ``distillation.distillmodel.KDModel`` and
``config.train_criterion`` a dict of losses weighted by ``config.loss_ratio``.  Every epoch evaluates the teacher and the
student; ``best_teacher.pth`` / ``best_student.pth`` follow each one's highest test acc1.  No EMA model, as in the
reference.
"""
import os

import torch

from .driver import Task, rename_if_exists, run
from .scripts import test_distill_classification, train_distill_classification
from .utils import unwrap


class DistillClassificationTask(Task):
    keep_ema = False

    def __init__(self):
        super().__init__(train_distill_classification, test_distill_classification)
        self.state = {'tea_best_acc1': 0., 'tea_test_loss': 0., 'stu_best_acc1': 0., 'stu_test_loss': 0.}

    def train_criterion(self, config):
        criterion = config.train_criterion
        for name in criterion:
            criterion[name] = criterion[name].cuda()
        return criterion

    def resume_info(self):
        s = self.state
        return f'tea_best_acc1 {s["tea_best_acc1"]:.3f}%, stu_best_acc1 {s["stu_best_acc1"]:.3f}%'

    def end_epoch(self, epoch, train_loss, result, model, eval_model, checkpoint_dir, config):
        tea_acc1, tea_acc5, tea_loss, stu_acc1, stu_acc5, stu_loss = result
        kd, s = unwrap(model), self.state
        s['tea_test_loss'], s['stu_test_loss'] = tea_loss, stu_loss
        for who, acc1, net in (('tea', tea_acc1, kd.teacher), ('stu', stu_acc1, kd.student)):
            if s[f'{who}_best_acc1'] < acc1 <= 100:
                s[f'{who}_best_acc1'] = acc1
                name = 'best_teacher.pth' if who == 'tea' else 'best_student.pth'
                torch.save(net.state_dict(), os.path.join(checkpoint_dir, name))   # no 'module.' prefix
        return (f'tea_acc1 {tea_acc1:.3f}%, tea_acc5 {tea_acc5:.3f}%, tea_test_loss {tea_loss:.4f}, '
                f'stu_acc1 {stu_acc1:.3f}%, stu_acc5 {stu_acc5:.3f}%, stu_test_loss {stu_loss:.4f}, ')

    def finish(self, checkpoint_dir, config):
        s = self.state
        rename_if_exists(checkpoint_dir, 'best_teacher.pth', f'teacher-epoch{config.epochs}-acc{s["tea_best_acc1"]:.3f}.pth')
        rename_if_exists(checkpoint_dir, 'best_student.pth', f'student-epoch{config.epochs}-acc{s["stu_best_acc1"]:.3f}.pth')


def main():
    run(DistillClassificationTask(), 'H100 distillation classification training')


if __name__ == '__main__':
    main()
