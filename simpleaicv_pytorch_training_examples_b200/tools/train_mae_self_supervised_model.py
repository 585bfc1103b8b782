"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_mae_self_supervised_model --work-dir DIR``

Drop-in for the reference's tools/train_mae_self_supervised_model.py (the three configs under
02.masked_image_modeling_training/imagenet/): ``config.model`` is a ``vit_*_mae_pretrain_model`` and the collater yields
the images and their patchified labels.  There is no test set: ``best.pth`` (the whole model) and ``best_encoder.pth``
(its encoder) follow the lowest epoch train loss, taken from the EMA model when there is one.
"""
import os

import torch

from .driver import Task, rename_if_exists, run
from .scripts import train_mae_self_supervised_learning
from .utils import unwrap


class MAETask(Task):

    def __init__(self):
        super().__init__(train_mae_self_supervised_learning)
        self.state = {'best_loss': 1e9, 'train_loss': 0.}

    def resume_info(self):
        return f'best_loss {self.state["best_loss"]:.4f}'

    def end_epoch(self, epoch, train_loss, result, model, eval_model, checkpoint_dir, config):
        self.state['train_loss'] = train_loss
        if train_loss < self.state['best_loss']:
            self.state['best_loss'] = train_loss
            net = unwrap(eval_model)
            torch.save(net.state_dict(), os.path.join(checkpoint_dir, 'best.pth'))
            torch.save(net.encoder.state_dict(), os.path.join(checkpoint_dir, 'best_encoder.pth'))
        return f'best_loss {self.state["best_loss"]:.4f}, '

    def finish(self, checkpoint_dir, config):
        best = self.state['best_loss']
        rename_if_exists(checkpoint_dir, 'best.pth', f'{config.network}-loss{best:.3f}.pth')
        rename_if_exists(checkpoint_dir, 'best_encoder.pth', f'{config.network}-loss{best:.3f}_encoder.pth')


def main():
    run(MAETask(), 'H100 MAE self-supervised training')


if __name__ == '__main__':
    main()
