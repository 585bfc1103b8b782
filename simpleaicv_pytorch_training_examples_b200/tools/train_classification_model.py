"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.train_classification_model --work-dir DIR``

Drop-in for the reference's tools/train_classification_model.py:33-283: reads ``config`` from
``<work-dir>/train_config.py`` (the same python-class config; only its ``backbones`` / ``losses``
imports point at this package), builds loaders / optimizer / scheduler, wraps the model for data
parallelism, resumes from ``checkpoints/latest.pth``, trains and evaluates every epoch and saves
``latest.pth`` / ``best.pth`` with the reference's checkpoint keys.  ``main(train_fn, test_fn)`` is shared by the entry
points whose epoch bodies differ (train_imagenet21k_classification_model); ``test_fn`` returns (acc1, acc5, loss) or
(acc1, loss).
"""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist
from torch.utils.data import DataLoader

from .scripts import test_classification, train_classification
from .utils import (Scheduler, build_optimizer, build_training_mode, checkpoint_model_state, get_logger, load_model_state,
                    set_seed, unwrap)


def parse_args():
    parser = argparse.ArgumentParser(description='H100 classification training')
    parser.add_argument('--work-dir', type=str, required=True, help='directory holding train_config.py')
    return parser.parse_args()


def main(train_fn=train_classification, test_fn=test_classification):
    assert torch.cuda.is_available(), 'need at least one H100 to train'
    args = parse_args()
    sys.path.append(args.work_dir)
    from train_config import config
    log_dir = os.path.join(args.work_dir, 'log')
    checkpoint_dir = os.path.join(args.work_dir, 'checkpoints')
    resume_model = os.path.join(checkpoint_dir, 'latest.pth')
    set_seed(config.seed)

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
    master = local_rank == 0 and int(os.environ.get('RANK', 0)) == 0
    if master:
        os.makedirs(checkpoint_dir, exist_ok=True)
        os.makedirs(log_dir, exist_ok=True)
    if dist.is_initialized():
        dist.barrier(device_ids=[local_rank])
    logger = get_logger('train', log_dir)

    batch_size = int(config.batch_size // world)       # config.batch_size is the global batch
    num_workers = max(1, int(config.num_workers // world))
    train_sampler = torch.utils.data.distributed.DistributedSampler(config.train_dataset, shuffle=True) if world > 1 else None
    train_loader = DataLoader(config.train_dataset, batch_size=batch_size, shuffle=train_sampler is None, pin_memory=True,
                              drop_last=True, num_workers=num_workers, collate_fn=config.train_collater, sampler=train_sampler)
    test_sampler = torch.utils.data.distributed.DistributedSampler(config.test_dataset, shuffle=False) if world > 1 else None
    test_loader = DataLoader(config.test_dataset, batch_size=batch_size, shuffle=False, pin_memory=True,
                             num_workers=num_workers, collate_fn=config.test_collater, sampler=test_sampler)

    model = config.model.cuda()
    train_criterion = config.train_criterion.cuda()
    test_criterion = config.test_criterion.cuda()
    optimizer, group_info = build_optimizer(config, model)
    scheduler = Scheduler(config, optimizer)
    model, config.ema_model, config.scaler = build_training_mode(config, model)
    if master:
        for k, v in config.__dict__.items():
            if not k.startswith('__') and k not in ('model',):
                logger.info(f'{k}: {v}')

    start_epoch, best_acc1, train_time = 1, 0., 0.
    if os.path.exists(resume_model):
        ckpt = torch.load(resume_model, map_location='cpu', weights_only=True)
        load_model_state(model, ckpt['model_state_dict'])
        optimizer.load_state_dict(ckpt['optimizer_state_dict'])
        scheduler.load_state_dict(ckpt['scheduler_state_dict'])
        if config.ema_model is not None and 'ema_model_state_dict' in ckpt:
            config.ema_model.ema_model.load_state_dict(ckpt['ema_model_state_dict'])
        start_epoch, best_acc1, train_time = ckpt['epoch'] + 1, ckpt['best_acc1'], ckpt.get('time', 0.)
        logger.info(f'resumed from epoch {ckpt["epoch"]:0>3d}, best_acc1 {best_acc1:.3f}%') if master else None

    for epoch in range(start_epoch, config.epochs + 1):
        t0 = time.time()
        if train_sampler is not None:
            train_sampler.set_epoch(epoch)
        train_loss = train_fn(train_loader, model, train_criterion, optimizer, scheduler, epoch, logger, config)
        eval_model = config.ema_model.ema_model if config.ema_model is not None else model
        result = test_fn(test_loader, eval_model, test_criterion, config)
        acc1, test_loss = result[0], result[-1]
        acc5 = f'acc5 {result[1]:.3f}%, ' if len(result) == 3 else ''
        train_time += (time.time() - t0) / 3600
        if master:
            logger.info(f'epoch {epoch:0>3d}: train loss {train_loss:.4f}, acc1 {acc1:.3f}%, {acc5}'
                        f'test loss {test_loss:.4f}, {(time.time() - t0) / 3600:.3f} h')
            if best_acc1 < acc1 <= 100:
                best_acc1 = acc1
                torch.save(unwrap(eval_model).state_dict(), os.path.join(checkpoint_dir, 'best.pth'))   # no 'module.' prefix
            state = {'epoch': epoch, 'time': train_time, 'best_acc1': best_acc1, 'test_loss': test_loss,
                     'lr': scheduler.current_lr, 'model_state_dict': checkpoint_model_state(model),   # 'module.'-prefixed
                     'optimizer_state_dict': optimizer.state_dict(), 'scheduler_state_dict': scheduler.state_dict()}
            if config.ema_model is not None:
                state['ema_model_state_dict'] = config.ema_model.ema_model.state_dict()
            torch.save(state, os.path.join(checkpoint_dir, 'latest.pth'))
    if master and os.path.exists(os.path.join(checkpoint_dir, 'best.pth')):
        os.rename(os.path.join(checkpoint_dir, 'best.pth'),
                  os.path.join(checkpoint_dir, f'{config.network}-acc{best_acc1:.3f}.pth'))
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
