"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_classification_model --work-dir DIR``

Drop-in for the reference's tools/train_classification_model.py:33-283: reads ``config`` from
``<work-dir>/train_config.py`` (the same python-class config; only its ``backbones`` / ``losses``
imports point at this package), builds loaders / optimizer / scheduler, wraps the model for data
parallelism, resumes from ``checkpoints/latest.pth``, trains and evaluates every epoch and saves
``latest.pth`` / ``best.pth`` with the reference's checkpoint keys.  ``main(train_fn, test_fn)`` is shared by the entry
points whose epoch bodies differ (train_imagenet21k_classification_model); ``test_fn`` returns (acc1, acc5, loss) or
(acc1, loss).  The loop itself is tools/driver.py.
"""
import os

import torch

from .driver import Task, rename_if_exists, run
from .scripts import test_classification, train_classification
from .utils import unwrap


class ClassificationTask(Task):
    """best.pth by the highest test acc1; latest.pth carries best_acc1 and test_loss."""

    def __init__(self, train_fn, test_fn):
        super().__init__(train_fn, test_fn)
        self.state = {'best_acc1': 0., 'test_loss': 0.}

    def resume_info(self):
        return f'best_acc1 {self.state["best_acc1"]:.3f}%'

    def end_epoch(self, epoch, train_loss, result, model, eval_model, checkpoint_dir, config):
        acc1, test_loss = result[0], result[-1]
        acc5 = f'acc5 {result[1]:.3f}%, ' if len(result) == 3 else ''
        self.state['test_loss'] = test_loss
        if self.state['best_acc1'] < acc1 <= 100:
            self.state['best_acc1'] = acc1
            torch.save(unwrap(eval_model).state_dict(), os.path.join(checkpoint_dir, 'best.pth'))   # no 'module.' prefix
        return f'acc1 {acc1:.3f}%, {acc5}test loss {test_loss:.4f}, '

    def finish(self, checkpoint_dir, config):
        rename_if_exists(checkpoint_dir, 'best.pth', f'{config.network}-acc{self.state["best_acc1"]:.3f}.pth')


def main(train_fn=train_classification, test_fn=test_classification):
    run(ClassificationTask(train_fn, test_fn), 'H100 classification training')


if __name__ == '__main__':
    main()
