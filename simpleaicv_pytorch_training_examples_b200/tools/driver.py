"""The training loop every ``tools/train_*_model`` entry point shares (the reference repeats it in each of its
tools/train_*_model.py): ``<work-dir>/train_config.py``, the process group, samplers and loaders from the global
``batch_size`` / ``num_workers``, the logger, ``build_optimizer``, ``Scheduler``, ``build_training_mode``, resume from
``checkpoints/latest.pth`` and one ``latest.pth`` per epoch.  A ``Task`` supplies what differs between the entry points:
the epoch bodies, whether there is a test set, the best-checkpoint rule, the files written and the extra ``latest.pth``
keys."""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist
from torch.utils.data import DataLoader

from .utils import (Scheduler, build_optimizer, build_training_mode, checkpoint_model_state, get_logger, load_model_state,
                    set_seed)


def parse_args(description):
    parser = argparse.ArgumentParser(description=description)
    parser.add_argument('--work-dir', type=str, required=True, help='directory holding the config')
    return parser.parse_args()


def init_distributed(config):
    """Sets config.local_rank / gpus_type / gpus_num / group like the reference and joins the process group when
    launched by torchrun.  Returns (local_rank, world size, whether this is the master rank)."""
    local_rank = int(os.environ.get('LOCAL_RANK', 0))
    world = int(os.environ.get('WORLD_SIZE', 1))
    config.local_rank = local_rank
    config.gpus_type = torch.cuda.get_device_name()
    config.gpus_num = world
    torch.cuda.set_device(local_rank)
    if world > 1 or 'RANK' in os.environ:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group(backend='nccl', init_method='env://', device_id=torch.device('cuda', local_rank))
    config.group = None  # scalars ride on the default communicator (one collective per step)
    return local_rank, world, local_rank == 0 and int(os.environ.get('RANK', 0)) == 0


def make_loader(config, dataset, collater, world, train):
    """A rank's loader: its share of the global config.batch_size / config.num_workers, a DistributedSampler at N > 1."""
    sampler = torch.utils.data.distributed.DistributedSampler(dataset, shuffle=train) if world > 1 else None
    loader = DataLoader(dataset, batch_size=int(config.batch_size // world), shuffle=train and sampler is None,
                        pin_memory=True, drop_last=train, num_workers=max(1, int(config.num_workers // world)),
                        collate_fn=collater, sampler=sampler)
    return loader, sampler


def log_config(logger, config):
    for k, v in config.__dict__.items():
        if not k.startswith('__') and k not in ('model',):
            logger.info(f'{k}: {v}')


class Task:
    """What one entry point adds to the shared loop.

    ``state`` holds the entry point's extra ``latest.pth`` keys with their starting values; ``run`` restores them on
    resume and writes them every epoch.  ``test_fn`` None means the task has no test set (no test loader and no
    ``test_criterion`` are built).  ``keep_ema`` False: the entry point has no EMA model, as the reference's distillation
    entry points, and a config asking for one is refused."""

    keep_ema = True

    def __init__(self, train_fn, test_fn=None):
        self.train_fn, self.test_fn = train_fn, test_fn
        self.state = {}

    def check(self, config):
        """Refuses, before anything is built, a config asking for what the entry point does not do."""
        if not self.keep_ema and getattr(config, 'use_ema_model', False):
            raise ValueError('this entry point trains without an EMA model: set use_ema_model = False in the config')

    def train_criterion(self, config):
        return config.train_criterion.cuda()

    def resume_info(self):
        """The part of the resume log line after the epoch."""
        raise NotImplementedError

    def end_epoch(self, epoch, train_loss, result, model, eval_model, checkpoint_dir, config):
        """Master rank only, after each epoch: updates ``state``, writes the best / per-epoch files and returns the part
        of the epoch log line between the train loss and the time.  ``result`` is what ``test_fn`` returned (None without
        a test set); ``eval_model`` is the EMA model when there is one, else ``model``."""
        raise NotImplementedError

    def finish(self, checkpoint_dir, config):
        """Master rank only, after the last epoch: renames the best files as the reference does."""


def rename_if_exists(checkpoint_dir, src, dst):
    if os.path.exists(os.path.join(checkpoint_dir, src)):
        os.rename(os.path.join(checkpoint_dir, src), os.path.join(checkpoint_dir, dst))


def run(task, description):
    assert torch.cuda.is_available(), 'need at least one H100 to train'
    args = parse_args(description)
    sys.path.append(args.work_dir)
    from train_config import config
    task.check(config)
    log_dir = os.path.join(args.work_dir, 'log')
    checkpoint_dir = os.path.join(args.work_dir, 'checkpoints')
    resume_model = os.path.join(checkpoint_dir, 'latest.pth')
    set_seed(config.seed)

    local_rank, world, master = init_distributed(config)
    if master:
        os.makedirs(checkpoint_dir, exist_ok=True)
        os.makedirs(log_dir, exist_ok=True)
    if dist.is_initialized():
        dist.barrier(device_ids=[local_rank])
    logger = get_logger('train', log_dir)

    train_loader, train_sampler = make_loader(config, config.train_dataset, config.train_collater, world, train=True)
    test_loader = test_criterion = None
    if task.test_fn is not None:
        test_loader, _ = make_loader(config, config.test_dataset, config.test_collater, world, train=False)

    model = config.model.cuda()
    train_criterion = task.train_criterion(config)
    if task.test_fn is not None:
        test_criterion = config.test_criterion.cuda()
    optimizer, group_info = build_optimizer(config, model)
    scheduler = Scheduler(config, optimizer)
    model, config.ema_model, config.scaler = build_training_mode(config, model)
    if master:
        log_config(logger, config)

    start_epoch, train_time = 1, 0.
    if os.path.exists(resume_model):
        ckpt = torch.load(resume_model, map_location='cpu', weights_only=True)
        load_model_state(model, ckpt['model_state_dict'])
        optimizer.load_state_dict(ckpt['optimizer_state_dict'])
        scheduler.load_state_dict(ckpt['scheduler_state_dict'])
        if config.ema_model is not None and 'ema_model_state_dict' in ckpt:
            config.ema_model.ema_model.load_state_dict(ckpt['ema_model_state_dict'])
        start_epoch, train_time = ckpt['epoch'] + 1, ckpt.get('time', 0.)
        task.state = {k: ckpt[k] for k in task.state}
        logger.info(f'resumed from epoch {ckpt["epoch"]:0>3d}, {task.resume_info()}') if master else None

    for epoch in range(start_epoch, config.epochs + 1):
        t0 = time.time()
        if train_sampler is not None:
            train_sampler.set_epoch(epoch)
        train_loss = task.train_fn(train_loader, model, train_criterion, optimizer, scheduler, epoch, logger, config)
        eval_model = config.ema_model.ema_model if config.ema_model is not None else model
        result = task.test_fn(test_loader, eval_model, test_criterion, config) if task.test_fn is not None else None
        train_time += (time.time() - t0) / 3600
        if master:
            info = task.end_epoch(epoch, train_loss, result, model, eval_model, checkpoint_dir, config)
            logger.info(f'epoch {epoch:0>3d}: train loss {train_loss:.4f}, {info}{(time.time() - t0) / 3600:.3f} h')
            state = {'epoch': epoch, 'time': train_time, **task.state,
                     'lr': scheduler.current_lr, 'model_state_dict': checkpoint_model_state(model),   # 'module.'-prefixed
                     'optimizer_state_dict': optimizer.state_dict(), 'scheduler_state_dict': scheduler.state_dict()}
            if config.ema_model is not None:
                state['ema_model_state_dict'] = config.ema_model.ema_model.state_dict()
            torch.save(state, os.path.join(checkpoint_dir, 'latest.pth'))
    if master:
        task.finish(checkpoint_dir, config)
    if dist.is_initialized():
        dist.destroy_process_group()
