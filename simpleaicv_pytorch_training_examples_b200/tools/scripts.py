"""train / test loops of the classification task with the call signatures of the reference's
tools/scripts.py:36-113 (test_classification), :116-275 (train_classification) and :1774-1934 (train_mae_self_supervised_learning),
and of tools/train_imagenet21k_classification_model.py:27-237 (ImageNet-21K semantic-softmax training).

Arithmetic per step is the reference's: forward, criterion, backward (gradient average across
ranks), optional clipping, optimizer step, per-iteration LR.  Control flow is tightened for the
GPU: the NaN/Inf guards are evaluated on the device and travel, together with the loss, in ONE
small all-reduce and ONE device->host read per step; there is no per-step barrier.
"""
import torch
import torch.distributed as dist

from ..classification.common import AccMeter, AverageMeter, SemanticSoftmaxMeter
from ..classification.semantic import SemanticTree


def _world():
    return dist.get_world_size() if dist.is_initialized() else 1


def all_reduce_operation_in_group_for_variables(variables, operator, group):
    """tools/scripts.py:26-33, but all scalars share one tensor / one collective / one sync."""
    t = torch.tensor([float(v) for v in variables], device='cuda', dtype=torch.float64)
    if dist.is_initialized() and _world() > 1:
        dist.all_reduce(t, op=operator, group=group)
    return t.tolist()


def _is_master(config):
    return config.local_rank == 0 and getattr(config, 'total_rank', 0) == 0


def train_classification(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute_loss=None):
    """compute_loss(model, criterion, images, labels) -> loss overrides the default criterion(model(images), labels): the
    epoch bodies of the reference that differ only there (train_mae_self_supervised_learning) share this loop."""
    losses = AverageMeter()
    model.train()
    accum = config.accumulation_steps
    assert accum >= 1, 'illegal accumulation_steps!'
    iters = len(train_loader.dataset) // config.batch_size
    group = getattr(config, 'group', None)
    world = _world()
    iter_index = 1
    from .utils import CudaPrefetcher
    # config.device_normalize = (mean, std): uint8 [B, H, W, 3] batches (classification.common.Uint8ClassificationCollater)
    # are normalised on the device by the prefetcher (SURVEY.md 8 f3); fp32 batches pass through unchanged
    for _, data in enumerate(CudaPrefetcher(train_loader, normalize=getattr(config, 'device_normalize', None))):
        images, labels = data['image'], data['label']
        bad = (~torch.isfinite(images)).any()
        if labels.dtype.is_floating_point:
            bad = bad | (~torch.isfinite(labels)).any()
        if compute_loss is not None:
            loss = compute_loss(model, criterion, images, labels)
        else:
            outputs = model(images)
            loss = criterion(outputs, labels)
        bad = bad | (~torch.isfinite(loss)) | (loss == 0.)
        loss = loss / accum
        sync_step = iter_index % accum == 0
        if sync_step or not hasattr(model, 'no_sync'):
            loss.backward()
        else:
            with model.no_sync():
                loss.backward()
        if getattr(config, 'skip_inf_nan_grad', False):
            for p in model.parameters():
                if p.grad is not None:
                    bad = bad | (~torch.isfinite(p.grad)).any()
        stat = torch.stack([bad.float(), loss.detach().float()])
        if world > 1:
            dist.all_reduce(stat, op=dist.ReduceOp.SUM, group=group)
        skip_count, loss_sum = stat.tolist()  # the one host sync of the step
        if skip_count > 0:
            logger.info('skip this batch!') if _is_master(config) else None
            optimizer.zero_grad()
            continue
        if sync_step:
            if getattr(config, 'clip_grad_value', 0) and config.clip_grad_value > 0:
                torch.nn.utils.clip_grad_value_(model.parameters(), config.clip_grad_value)
            if getattr(config, 'clip_max_norm', 0) and config.clip_max_norm > 0:
                if hasattr(optimizer, 'clip_grad_norm'):    # fused: coefficient stays on the device, applied inside step()
                    optimizer.clip_grad_norm(config.clip_max_norm)
                else:
                    torch.nn.utils.clip_grad_norm_(model.parameters(), config.clip_max_norm)
            optimizer.step()
            optimizer.zero_grad()
            if getattr(config, 'use_ema_model', False):
                config.ema_model.update(model)
            loss_value = loss_sum / world
            losses.update(loss_value, images.size(0))
            scheduler.step(optimizer, iter_index / iters + (epoch - 1))
        if iter_index % int(config.print_interval * accum) == 0 and _is_master(config):
            logger.info(f'train: epoch {epoch:0>4d}, iter [{iter_index // accum:0>5d}, {iters // accum:0>5d}], '
                        f'lr: {scheduler.current_lr:.6f}, loss: {loss_sum / world * accum:.4f}')
        iter_index += 1
    return losses.avg * accum


def train_mae_self_supervised_learning(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config):
    """tools/scripts.py:1774-1934 of the reference: `outputs, masks = model(images); loss = criterion(outputs, labels, masks)`
    with the guards / accumulation / clipping / per-iteration LR of train_classification (labels = patchified images)."""
    def mae_loss(model, criterion, images, labels):
        outputs, masks = model(images)
        return criterion(outputs, labels, masks)
    return train_classification(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute_loss=mae_loss)


def train_imagenet21k_classification(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config):
    """tools/train_imagenet21k_classification_model.py:94-237 of the reference: `criterion(semantic outputs, semantic labels)`
    with the guards / accumulation / clipping / per-iteration LR of train_classification.  The tree of config.train_dataset
    is built once; label conversion is a device gather, so the step keeps its one host sync."""
    tree = SemanticTree.of(config.train_dataset)

    def semantic_loss(model, criterion, images, labels):
        outputs = model(images)
        return criterion(tree.convert_outputs_to_semantic_outputs(outputs), tree.convert_single_labels_to_semantic_labels(labels))
    return train_classification(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config,
                                compute_loss=semantic_loss)


def train_epoch_with_loss_terms(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute,
                                total_name='total_loss'):
    """Shared epoch body of the reference's dict-loss training loops (train_detection, tools/scripts.py:900-1092;
    train_distill_sam_encoder, tools/interactive_segmentation_scripts.py:21-199): `compute(data)` runs the model and the
    criterion on one device-resident batch and returns (dict of loss terms, tensors to check for inf / nan, batch size).
    NaN / inf / zero-loss guards skip the batch on every rank; accumulation under no_sync(); clipping; per-iteration LR.
    The reference all-reduces the skip flag, every loss term and the total with one host sync each (>= 20 per step for
    DETR's 18 terms); here they travel in ONE coalesced all-reduce and are read with one sync."""
    losses = AverageMeter()
    accum = config.accumulation_steps
    assert accum >= 1, 'illegal accumulation_steps!'
    iters = len(train_loader.dataset) // config.batch_size
    group = getattr(config, 'group', None)
    world = _world()
    iter_index = 1
    from .utils import CudaPrefetcher
    # config.device_normalize = (mean, std): uint8 [B, H, W, 3] batches (classification.common.Uint8ClassificationCollater)
    # are normalised on the device by the prefetcher (SURVEY.md 8 f3); fp32 batches pass through unchanged
    for _, data in enumerate(CudaPrefetcher(train_loader, normalize=getattr(config, 'device_normalize', None))):
        loss_value, checked, batch = compute(data)
        bad = torch.zeros((), dtype=torch.bool, device=next(iter(loss_value.values())).device)
        for t in checked:
            bad = bad | (~torch.isfinite(t)).any()
        names = list(loss_value)
        terms = torch.stack([loss_value[k].float() for k in names])
        loss = terms.sum()
        bad = bad | (~torch.isfinite(terms)).any() | (loss == 0.)
        loss = loss / accum
        sync_step = iter_index % accum == 0
        if sync_step or not hasattr(model, 'no_sync'):
            loss.backward()
        else:
            with model.no_sync():
                loss.backward()
        if getattr(config, 'skip_inf_nan_grad', False):
            for p in model.parameters():
                if p.grad is not None:
                    bad = bad | (~torch.isfinite(p.grad)).any()
        stat = torch.cat([bad.float().view(1), loss.detach().float().view(1), terms.detach() / accum])
        if world > 1:
            dist.all_reduce(stat, op=dist.ReduceOp.SUM, group=group)
        stat = stat.tolist()  # the one host sync of the step
        skip_count, loss_sum, term_sums = stat[0], stat[1], stat[2:]
        if skip_count > 0:
            logger.info('skip this batch!') if _is_master(config) else None
            optimizer.zero_grad()
            continue
        if sync_step:
            if getattr(config, 'clip_grad_value', 0) and config.clip_grad_value > 0:
                torch.nn.utils.clip_grad_value_(model.parameters(), config.clip_grad_value)
            if getattr(config, 'clip_max_norm', 0) and config.clip_max_norm > 0:
                if hasattr(optimizer, 'clip_grad_norm'):    # fused: coefficient stays on the device, applied inside step()
                    optimizer.clip_grad_norm(config.clip_max_norm)
                else:
                    torch.nn.utils.clip_grad_norm_(model.parameters(), config.clip_max_norm)
            optimizer.step()
            optimizer.zero_grad()
            if getattr(config, 'use_ema_model', False):
                config.ema_model.update(model)
            losses.update(loss_sum / world, batch)
            scheduler.step(optimizer, iter_index / iters + (epoch - 1))
        if iter_index % int(config.print_interval * accum) == 0 and _is_master(config):
            msg = (f'train: epoch {epoch:0>4d}, iter [{iter_index // accum:0>5d}, {iters // accum:0>5d}], lr: {scheduler.current_lr:.6f}, '
                   f'{total_name}: {loss_sum / world * accum:.4f}, ')
            msg += ''.join(f'{k}: {v / world * accum:.4f}, ' for k, v in zip(names, term_sums))
            logger.info(msg)
        iter_index += 1
    return losses.avg * accum


def train_distill_classification(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config):
    """tools/scripts.py:291-500 of the reference: `tea_outputs, stu_outputs = model(images)`; `criterion` is a dict of
    losses, CELoss / OneHotLabelCELoss apply to the student (and to the teacher when it is not frozen), every other entry
    to (student, teacher); each term is weighted by config.loss_ratio[name]; the frozen teacher stays in eval mode."""
    model.train()
    if config.freeze_teacher:
        (model.module if hasattr(model, 'module') else model).teacher.eval()

    def compute(data):
        images, labels = data['image'], data['label']
        tea_outputs, stu_outputs = model(images)
        loss_value = {}
        for name, fn in criterion.items():
            if name in ('CELoss', 'OneHotLabelCELoss'):
                if not config.freeze_teacher:
                    loss_value['tea_' + name] = fn(tea_outputs, labels) * config.loss_ratio[name]
                loss_value['stu_' + name] = fn(stu_outputs, labels) * config.loss_ratio[name]
            else:
                loss_value[name] = fn(stu_outputs, tea_outputs) * config.loss_ratio[name]
        checked = (images, labels) if labels.dtype.is_floating_point else (images,)
        return loss_value, checked, images.size(0)

    return train_epoch_with_loss_terms(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute,
                                       total_name='loss')


def train_detection(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config):
    """One epoch of detection training with the reference's step semantics (tools/scripts.py:900-1092): DETR batches carry
    'image', 'scaled_annots' and 'mask'; the criterion returns a dict of loss terms whose sum is differentiated."""
    model.train()
    is_detr = 'detr' in config.network

    def compute(data):
        images = data['image']
        targets = data['scaled_annots'] if is_detr else data['annots']
        outs = model(images, data['mask']) if is_detr else model(images)
        return criterion(outs, targets), (images, targets), images.size(0)

    return train_epoch_with_loss_terms(train_loader, model, criterion, optimizer, scheduler, epoch, logger, config, compute)


def _eval_batches(test_loader, config):
    """config.device_normalize = (mean, std): the batches go through CudaPrefetcher, so uint8 ones (Uint8Resize +
    Uint8CenterCrop + Uint8ClassificationCollater) are resized and normalised on the device; fp32 ones pass unchanged."""
    normalize = getattr(config, 'device_normalize', None)
    if normalize is None:
        return test_loader
    from .utils import CudaPrefetcher
    return CudaPrefetcher(test_loader, normalize=normalize)


@torch.no_grad()
def test_classification(test_loader, model, criterion, config):
    """Returns (acc1 %, acc5 %, loss); top-k indices come from torch.topk like the reference
    (tools/scripts.py:74-95) so index ties resolve identically."""
    model.eval()
    group = getattr(config, 'group', None)
    meter = AccMeter()
    loss_sum = 0.
    for data in _eval_batches(test_loader, config):
        images, labels = data['image'].cuda(non_blocking=True), data['label'].cuda(non_blocking=True)
        outputs = model(images)
        loss = criterion(outputs, labels)
        _, pred = torch.topk(outputs.float(), k=5, dim=1, largest=True, sorted=True)
        pred = pred.t()
        hit = pred.eq(labels.view(1, -1).expand_as(pred))
        meter.update(hit[:1].reshape(-1).float().sum().item(), hit[:5].reshape(-1).float().sum().item(), images.size(0))
        loss_sum += loss.item() * images.size(0)
    meter.acc1_correct_num, meter.acc5_correct_num, meter.sample_num, loss_sum = all_reduce_operation_in_group_for_variables(
        [meter.acc1_correct_num, meter.acc5_correct_num, meter.sample_num, loss_sum], dist.ReduceOp.SUM, group)
    meter.compute()
    return meter.acc1 * 100, meter.acc5 * 100, loss_sum / meter.sample_num


@torch.no_grad()
def test_imagenet21k_classification(test_loader, model, criterion, config):
    """tools/train_imagenet21k_classification_model.py:27-91 of the reference: returns (acc1 %, mean loss) over the semantic
    levels (SemanticSoftmaxMeter).  Loss and accuracy counts accumulate on the device and cross the host, and the ranks, in
    one all-reduce at the end of the evaluation."""
    model.eval()
    tree = SemanticTree.of(config.test_dataset)
    group = getattr(config, 'group', None)
    accs = SemanticSoftmaxMeter()
    loss_sum, samples = 0., 0
    for data in _eval_batches(test_loader, config):
        images, labels = data['image'].cuda(non_blocking=True), data['label'].cuda(non_blocking=True)
        outputs = tree.convert_outputs_to_semantic_outputs(model(images))
        labels = tree.convert_single_labels_to_semantic_labels(labels)
        loss_sum = loss_sum + criterion(outputs, labels).detach().double() * images.size(0)
        accs.update_per_batch(*accs.compute_per_batch(outputs, labels))
        samples += images.size(0)
    accs.sum, accs.count, loss_sum, samples = all_reduce_operation_in_group_for_variables(
        [accs.sum, accs.count, loss_sum, samples], dist.ReduceOp.SUM, group)
    accs.compute()
    return accs.acc1 * 100, (loss_sum / samples if samples else 0.)
