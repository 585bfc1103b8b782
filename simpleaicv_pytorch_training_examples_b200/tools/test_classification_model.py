"""``torchrun --nproc_per_node=N -m simpleaicv_pytorch_training_examples_b200.tools.test_classification_model --work-dir DIR``

Drop-in for the reference's tools/test_classification_model.py, the tool the classification configs' ``test.sh`` calls:
reads ``config`` from ``<work-dir>/test_config.py`` (the config loads its own weights into ``config.model``), evaluates it
with ``scripts.test_classification`` over ``config.test_dataset`` and logs acc1, acc5 and the test loss to
``<work-dir>/log/test.info.log``.  The log names the parameter count instead of the reference's FLOPs / MACs (which need
``calflops``), and there are no per-image load / inference times (test_classification does not measure them).
"""
import sys

import torch
import torch.distributed as dist

from .driver import init_distributed, log_config, make_loader, parse_args
from .scripts import test_classification
from .utils import get_logger, set_seed


def main():
    assert torch.cuda.is_available(), 'need at least one H100 to test'
    args = parse_args('H100 classification testing')
    sys.path.append(args.work_dir)
    from test_config import config
    set_seed(config.seed)
    local_rank, world, master = init_distributed(config)
    logger = get_logger('test', f'{args.work_dir}/log')
    test_loader, _ = make_loader(config, config.test_dataset, config.test_collater, world, train=False)
    if master:
        log_config(logger, config)
    model = config.model
    params = sum(p.numel() for p in model.parameters())
    logger.info(f'model: {config.network}, params: {params}') if master else None
    model = model.cuda()
    acc1, acc5, test_loss = test_classification(test_loader, model, config.test_criterion.cuda(), config)
    logger.info(f'acc1: {acc1:.3f}%, acc5: {acc5:.3f}%, test_loss: {test_loss:.4f}') if master else None
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
