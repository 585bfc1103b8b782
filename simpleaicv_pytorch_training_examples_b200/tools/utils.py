"""Host-side helpers with the semantics of the reference's tools/utils.py, for the H100 path.

  get_logger            tools/utils.py:66-92   (rank-0 file + stderr logging)
  set_seed              tools/utils.py:95-107
  build_optimizer       tools/utils.py:292-680 (param groups by weight decay / lr / layer decay; Muon split)
  Scheduler             tools/utils.py:205-289 (per-iteration MultiStep / Cosine / Poly LR, warm-up)
  build_training_mode   tools/utils.py:175-202 (DDP wrap -> distributed.B200DataParallel)
  EmaModel              tools/utils.py:145-172
"""
import copy
import logging
import math
import os
import random
from logging.handlers import TimedRotatingFileHandler

import numpy as np
import torch


def get_logger(name, log_dir):
    logger = logging.getLogger(name)
    logger.setLevel(logging.INFO)
    if logger.handlers:
        return logger
    os.makedirs(log_dir, exist_ok=True)
    fmt = logging.Formatter('%(asctime)s - %(levelname)s - %(message)s')
    fh = TimedRotatingFileHandler(os.path.join(log_dir, f'{name}.info.log'), when='W0', encoding='utf-8')
    fh.setLevel(logging.INFO)
    fh.setFormatter(fmt)
    sh = logging.StreamHandler()
    sh.setLevel(logging.INFO)
    sh.setFormatter(fmt)
    logger.addHandler(fh)
    logger.addHandler(sh)
    return logger


def set_seed(seed):
    """Seeds python / numpy / torch (CPU + CUDA) like the reference.  The reference also forces
    deterministic cuDNN; the H100 path does not use cuDNN, so there is nothing to pin there."""
    random.seed(seed)
    np.random.seed(seed)
    os.environ['PYTHONHASHSEED'] = str(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)
        torch.cuda.manual_seed_all(seed)


def _first_match(table, name, default):
    if isinstance(table, dict):
        for key, value in table.items():
            if key in name:
                return value
    return default


def param_group_table(config, model):
    """Returns [{'name', 'param', 'weight_decay', 'lr', 'lr_scale'}] for every trainable
    parameter, following the rules of tools/utils.py:292-600:
      * global_weight_decay False -> 1-D params and names matching no_weight_decay_layer_name_list
        get weight decay 0; 'sub_layer_weight_decay' / 'sub_layer_lr' override by name substring;
      * ViT layer-wise lr decay ('lr_layer_decay', 'lr_layer_decay_block', 'block_name'): scale
        lr_layer_decay**(L+1-i) for block i, lr_layer_decay**(L+1) for position/cls/patch
        embeddings, 1 for the rest."""
    opt = config.optimizer[1]
    lr, wd = opt['lr'], opt['weight_decay']
    global_wd = opt.get('global_weight_decay', True)
    no_wd_names = opt.get('no_weight_decay_layer_name_list', []) if isinstance(
        opt.get('no_weight_decay_layer_name_list', []), list) else []
    layer_decay = 'block_name' in opt
    rows = []
    if layer_decay:
        blocks = list(opt['lr_layer_decay_block'])
        num_layers = len(blocks) + 1
        scales = [opt['lr_layer_decay'] ** (num_layers - i) for i in range(num_layers + 1)]
        block_param_ids = [{id(p) for p in blk.parameters()} for blk in blocks]
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        if global_wd:
            decay = wd
        elif p.ndim == 1 or any(s in name for s in no_wd_names):
            decay = 0.
        else:
            decay = _first_match(opt.get('sub_layer_weight_decay'), name, wd)
        plr = _first_match(opt.get('sub_layer_lr'), name, lr)
        scale = 1.
        if layer_decay:
            if opt['block_name'] in name:
                idx = next(i for i, ids in enumerate(block_param_ids) if id(p) in ids)
                scale = scales[idx + 1]
            elif any(s in name for s in ('position_encoding', 'cls_token', 'patch_embedding')):
                scale = scales[0]
        rows.append({'name': name, 'param': p, 'weight_decay': decay, 'lr': plr, 'lr_scale': scale})
    return rows


MUON_EXCLUDE = ('position_encoding', 'cls_token', 'patch_embedding')


def muon_split(opt, model):
    """(muon [(name, param)], adamw [(name, param)], description list) of the trainable parameters for the optimizer
    config `opt`: Muon takes the >= 2-D ones whose name contains none of MUON_EXCLUDE + exclude_muon_layer_name_list
    (the reference's rule, tools/utils.py:609-655)."""
    extra = opt['exclude_muon_layer_name_list'] if isinstance(opt.get('exclude_muon_layer_name_list'), list) else []
    names = list(MUON_EXCLUDE) + extra
    muon, adamw = [], []
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        (muon if p.ndim >= 2 and not any(e in name for e in names) else adamw).append((name, p))
    info = [{'name': [n for n, _ in ps], 'optimizer': kind, 'lr': opt['lr'], 'weight_decay': opt['weight_decay']}
            for kind, ps in (('Muon', muon), ('AdamW', adamw)) if ps]
    return muon, adamw, info


def _build_muon(opt, model):
    """The reference's Muon branch: one lr / weight decay for every parameter (per-layer lr / wd, layer decay and
    no-weight-decay lists are ignored, as there)."""
    muon, adamw, info = muon_split(opt, model)
    lr, wd = opt['lr'], opt['weight_decay']
    from ..optim import FusedMuon   # raises a RuntimeError on CPU parameters: there is no CPU implementation
    optimizer = FusedMuon(lr=lr, wd=wd, muon_params=[p for _, p in muon], adamw_params=[p for _, p in adamw],
                          momentum=opt.get('momentum', 0.95), nesterov=opt.get('nesterov', True),
                          ns_steps=opt.get('ns_steps', 5),
                          adamw_betas=(opt.get('adamw_beta1', 0.9), opt.get('adamw_beta2', 0.999)),
                          adamw_eps=opt.get('adamw_eps', 1e-8)).attach(model)
    return optimizer, info


def build_optimizer(config, model):
    """Returns (optimizer, group description list) like the reference."""
    name, opt = config.optimizer
    assert name in ('SGD', 'AdamW', 'Muon'), 'Unsupported optimizer!'
    if name == 'Muon':
        return _build_muon(opt, model)
    rows = param_group_table(config, model)
    groups, descr = {}, {}
    for r in rows:
        key = (r['weight_decay'], r['lr'], r['lr_scale'])
        groups.setdefault(key, []).append(r['param'])
        descr.setdefault(key, []).append(r['name'])
    param_groups = [{'params': ps, 'weight_decay': k[0], 'lr': k[1] * k[2]} for k, ps in groups.items()]
    info = [{'name': descr[k], 'weight_decay': k[0], 'lr': k[1], 'lr_scale': k[2]} for k in groups]
    # fused multi-tensor step (optim.py, SURVEY.md 8 f2) whenever the parameters live on the GPU; 'fused': False in the
    # optimizer config keeps torch.optim (the reference's tools/utils.py:581-600)
    fused = bool(opt.get('fused', True)) and len(rows) > 0 and all(r['param'].is_cuda for r in rows)
    if name == 'SGD':
        if fused:
            from ..optim import FusedSGD
            optimizer = FusedSGD(param_groups, lr=opt['lr'], momentum=opt['momentum'], nesterov=opt.get('nesterov', False)).attach(model)
        else:
            optimizer = torch.optim.SGD(param_groups, lr=opt['lr'], momentum=opt['momentum'],
                                        nesterov=opt.get('nesterov', False))
    else:
        if fused:
            from ..optim import FusedAdamW
            optimizer = FusedAdamW(param_groups, lr=opt['lr'], betas=(opt.get('beta1', 0.9), opt.get('beta2', 0.999)),
                                   eps=opt.get('eps', 1e-8)).attach(model)
        else:
            optimizer = torch.optim.AdamW(param_groups, lr=opt['lr'], betas=(opt.get('beta1', 0.9), opt.get('beta2', 0.999)),
                                          eps=opt.get('eps', 1e-8), capturable=bool(opt.get('capturable', False)))
    return optimizer, info


class Scheduler:
    """Per-iteration learning-rate schedule: step(optimizer, fractional_epoch)."""

    def __init__(self, config, optimizer):
        self.scheduler_name, self.scheduler_parameters = config.scheduler
        assert self.scheduler_name in ('MultiStepLR', 'CosineLR', 'PolyLR'), 'Unsupported scheduler!'
        self.warm_up_epochs = self.scheduler_parameters['warm_up_epochs']
        self.epochs = config.epochs
        self.lr = config.optimizer[1]['lr']
        self.current_lr = self.lr
        self.init_param_groups_lr = [g['lr'] for g in optimizer.param_groups]
        assert self.warm_up_epochs >= 0 and self.epochs > 0

    def _factor(self, epoch, base):
        sp = self.scheduler_parameters
        if epoch < self.warm_up_epochs:
            return epoch / self.warm_up_epochs * base
        if self.scheduler_name == 'MultiStepLR':
            return sp['gamma'] ** len([m for m in sp['milestones'] if m <= epoch]) * base
        min_lr = sp.get('min_lr', 0.)
        t = (epoch - self.warm_up_epochs) / (self.epochs - self.warm_up_epochs)
        if self.scheduler_name == 'CosineLR':
            return 0.5 * (math.cos(t * math.pi) + 1) * (base - min_lr) + min_lr
        return ((1 - t) ** sp['power']) * (base - min_lr) + min_lr

    def step(self, optimizer, epoch):
        assert len(self.init_param_groups_lr) == len(optimizer.param_groups)
        for g, base in zip(optimizer.param_groups, self.init_param_groups_lr):
            g['lr'] = self._factor(epoch, base)
        self.current_lr = self._factor(epoch, self.lr)

    def state_dict(self):
        return dict(self.__dict__)

    def load_state_dict(self, state_dict):
        self.__dict__.update(state_dict)


class EmaModel:
    """Exponential moving average of the model's state_dict (off in the shipped hot-path configs)."""

    def __init__(self, model, decay=0.9999):
        self.ema_model = copy.deepcopy(model.module if hasattr(model, 'module') else model)
        self.decay = decay
        self.ema_model.eval()
        for p in self.ema_model.parameters():
            p.requires_grad_(False)

    @torch.no_grad()
    def update(self, model):
        src = (model.module if hasattr(model, 'module') else model).state_dict()
        for k, v in self.ema_model.state_dict().items():
            if v.dtype.is_floating_point:
                v.mul_(self.decay).add_(src[k].detach(), alpha=1. - self.decay)
            else:
                v.copy_(src[k])


class CudaPrefetcher:
    """Wraps a loader of {'image': pinned CPU tensor, 'label': ...} batches: the host->device copy
    of batch i+1 is issued on a side stream before the kernels of step i are enqueued, so PCIe
    traffic overlaps compute (the reference does a blocking ``.cuda()`` per step,
    tools/scripts.py:143).  Yields dicts of device tensors that are safe to use on the current
    stream.

    The device tensors live in TWO persistent slots that alternate (allocated on first use, re-allocated
    only when a batch changes shape): a fresh ``.to(device)`` per batch would go through the caching
    allocator on the side stream, whose cross-stream reuse rules can turn into cudaMalloc / cudaFree
    calls (device-wide syncs of several ms) in the middle of the step.  A slot is overwritten only after
    the consumer has asked for the following batch, i.e. after everything that reads it was enqueued:
    the side stream waits for an event recorded on the consumer's stream when it comes back for the next
    batch.  Consequently a yielded batch is valid until the consumer requests the next one (work already
    enqueued on the consumer's stream still sees the old contents; tensors to keep longer must be cloned)."""

    def __init__(self, loader, device=None, copy_streams=4, normalize=None):
        """normalize=(mean, std): batches whose 'image' is a uint8 [B, H, W, 3] tensor (classification.common.
        Uint8ClassificationCollater) are copied as uint8 - a quarter of the bytes - and turned into the fp32 NCHW
        normalised batch on the device, on the copy stream (SURVEY.md 8 f3; csrc/capi_input.cu).  Batches that also carry a
        'mixup' record (classification.common.Uint8MixupCutmixClassificationCollater) get the reference's RandomErasing and
        Mixup / CutMix applied by the same pass and are yielded as {'image': fp32 [B, 3, H, W], 'label': fp32 [B, classes]};
        such a batch without ``normalize`` raises.  When that record also holds RandAugment draws (classification.common.
        Uint8RandAugment), RandAugment is applied to the uint8 copy first, on the same stream.  Batches that carry a 'resample'
        ResampleBatch (samples from classification.common.Uint8RandomResizedCrop or Uint8Resize) copy the packed crops into
        a device buffer that only grows and resize them into the uint8 image first (ops.u8_resample), on the same stream.
        Batches that carry a 'resize_pad' ResizePadBatch (detection.common.Uint8DETRDetectionCollater, interactive_segmentation.
        common.Uint8SAMBatchCollater) copy their uint8 sources the same way and get the fp32 'image' - translated, resized,
        normalised as the record says and padded - and, for DETR, the bool padding 'mask' (ops.u8_resize_pad); they need no
        ``normalize``.
        copy_streams > 1: tensors of 32 MB and more are copied in that many chunks on separate streams, so that the copy of
        the next batch keeps its bandwidth while the current step's kernels run (tests/profile_h2d.py measures it)."""
        self.loader = loader
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else device
        self.stream = torch.cuda.Stream(self.device)
        self._extra = [torch.cuda.Stream(self.device) for _ in range(max(0, int(copy_streams) - 1))]
        self._slots = [{}, {}]
        self._free = [None, None]      # event after which slot k may be overwritten
        self.normalize = normalize

    def __len__(self):
        return len(self.loader)

    def _issue(self, it, k):
        batch = next(it, None)
        if batch is None:
            return None
        rec = batch.get('mixup')
        if rec is not None and self.normalize is None:
            raise RuntimeError("a batch with a 'mixup' record (Uint8MixupCutmixClassificationCollater) needs "
                               'CudaPrefetcher(normalize=(mean, std)): its uint8 pixels are not the model input')
        slot = self._slots[k & 1]
        with torch.cuda.stream(self.stream):
            if self._free[k & 1] is not None:
                self.stream.wait_event(self._free[k & 1])
            out = {}
            for name, v in batch.items():
                if name in ('mixup', 'resample', 'resize_pad'):
                    continue
                if not torch.is_tensor(v):
                    out[name] = v
                    continue
                buf = slot.get(name)
                if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                    buf = slot[name] = torch.empty(v.shape, dtype=v.dtype, device=self.device)
                self._copy(buf, v)
                out[name] = buf
            rs = batch.get('resample')
            rp = batch.get('resize_pad')
            packed = None
            if rs is not None or rp is not None:
                data = (rs if rs is not None else rp).data
                used = data.numel()
                packed = slot.get('resample_src')
                if packed is None or packed.numel() < used:
                    # the packed length changes every batch: the buffer only grows, to powers of two
                    packed = slot['resample_src'] = torch.empty(1 << max(used - 1, 0).bit_length(), dtype=torch.uint8,
                                                                device=self.device)
                packed = packed[:used]
                self._copy(packed, data)
            for st in self._extra:
                self.stream.wait_stream(st)
            if rp is not None:
                out['image'], mask = self._resize_pad(slot, packed, rp)
                if mask is not None:
                    out['mask'] = mask
            if rs is not None:
                from .. import ops
                shape = (rs.geom.shape[0],) + rs.out_hw + (3,)
                img = slot.get('resample_image')
                if img is None or tuple(img.shape) != shape:
                    img = slot['resample_image'] = torch.empty(shape, dtype=torch.uint8, device=self.device)
                out['image'] = ops.u8_resample(packed, rs.offsets, rs.geom, out=img)
            img = out.get('image')
            if self.normalize is not None and torch.is_tensor(img) and img.dtype == torch.uint8:
                from .. import ops
                nb = slot.get('image_f32')
                if nb is None or nb.shape[0] != img.shape[0] or nb.shape[2:] != img.shape[1:3]:
                    nb = slot['image_f32'] = torch.empty(img.shape[0], 3, img.shape[1], img.shape[2], device=self.device)
                if rec is None:
                    out['image'] = ops.u8_normalize(img, self.normalize[0], self.normalize[1], out=nb)
                else:
                    out['image'], out['label'] = self._mix(slot, img, out['label'], rec, nb)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return out, ev

    def _copy(self, buf, v):
        """buf.copy_(v) on the copy stream; 32 MB and more are split over the extra streams."""
        if self._extra and v.dim() > 0 and v.numel() * v.element_size() >= (32 << 20) and v.shape[0] >= len(self._extra) + 1:
            parts = len(self._extra) + 1
            step = (v.shape[0] + parts - 1) // parts
            buf[:step].copy_(v[:step], non_blocking=True)
            for j, st in enumerate(self._extra):
                st.wait_stream(self.stream)            # inherits the slot-free dependency
                with torch.cuda.stream(st):
                    lo = (j + 1) * step
                    buf[lo:lo + step].copy_(v[lo:lo + step], non_blocking=True)
        else:
            buf.copy_(v, non_blocking=True)

    def _resize_pad(self, slot, packed, rp):
        from .. import ops
        n, size = rp.geom.shape[0], rp.size
        img = slot.get('resize_pad_image')
        if img is None or tuple(img.shape) != (n, 3, size, size):
            img = slot['resize_pad_image'] = torch.empty(n, 3, size, size, device=self.device)
        mask = None
        if rp.with_mask:
            mask = slot.get('resize_pad_mask')
            if mask is None or tuple(mask.shape) != (n, size, size):
                mask = slot['resize_pad_mask'] = torch.empty(n, size, size, dtype=torch.bool, device=self.device)
        return ops.u8_resize_pad(packed, rp, out=img, mask=mask)

    def _mix(self, slot, img, labels, rec, out):
        from .. import ops
        if rec.randaug_ops is not None:
            scratch = slot.get('randaug_scratch')
            if scratch is None or scratch.shape != img.shape:
                scratch = slot['randaug_scratch'] = torch.empty_like(img)
                slot['randaug_stats'] = torch.empty(img.shape[0], 770, dtype=torch.int32, device=self.device)
            ops.u8_rand_augment(img, rec, scratch=scratch, stats=slot['randaug_stats'])
        used = rec.noise.numel()
        noise = slot.get('mixup_noise')
        if noise is None or noise.numel() < used:
            # the noise length changes every batch: the buffer only grows, to powers of two, so it is rarely re-allocated
            noise = slot['mixup_noise'] = torch.empty(1 << max(used - 1, 0).bit_length(), device=self.device)
        if used:
            noise[:used].copy_(rec.noise, non_blocking=True)
        soft = slot.get('mixup_label')
        if soft is None or tuple(soft.shape) != (img.shape[0], rec.num_classes):
            soft = slot['mixup_label'] = torch.empty(img.shape[0], rec.num_classes, device=self.device)
        return ops.u8_mix_erase_normalize(img, labels, self.normalize[0], self.normalize[1], rec, noise, out=out, soft=soft)

    def __iter__(self):
        it = iter(self.loader)
        k = 0
        nxt = self._issue(it, k)
        while nxt is not None:
            cur, ev = nxt
            main = torch.cuda.current_stream(self.device)
            main.wait_event(ev)
            k += 1
            nxt = self._issue(it, k)  # batch i+1 starts copying before step i is enqueued
            yield cur
            # the consumer is back: every kernel that reads `cur` has been enqueued on its stream
            done = torch.cuda.Event()
            done.record(torch.cuda.current_stream(self.device))
            self._free[(k - 1) & 1] = done


def unwrap(model):
    """The bare network under a data-parallel wrapper (torch DDP or B200DataParallel)."""
    return model.module if hasattr(model, 'module') else model


def checkpoint_model_state(model):
    """``model_state_dict`` of latest.pth in the REFERENCE's layout: the reference always saves the
    state_dict of the DDP-wrapped model (tools/train_classification_model.py:226-229), i.e. every key
    carries the ``module.`` prefix, whatever the world size.  best.pth holds ``unwrap(model).state_dict()``
    (no prefix, :213-221)."""
    return {'module.' + k: v for k, v in unwrap(model).state_dict().items()}


def load_model_state(model, state_dict, strict=True):
    """Loads a ``model_state_dict`` written by this package or by the reference, with or without the
    ``module.`` prefix, into a wrapped or unwrapped model (so runs can resume across 1 <-> N GPUs and
    from reference checkpoints)."""
    if state_dict and all(k.startswith('module.') for k in state_dict):
        state_dict = {k[len('module.'):]: v for k, v in state_dict.items()}
    return unwrap(model).load_state_dict(state_dict, strict=strict)


def build_training_mode(config, model):
    """Returns (model, ema_model, scaler).  The reference wraps in torch DDP and creates a
    GradScaler; here the wrapper is distributed.B200DataParallel (bucketed NCCL all-reduce fed
    directly by the runtime) and no GradScaler exists: the kernels compute in bf16 with fp32
    accumulation / statistics, which needs no loss scaling.

    sync_bn (the reference: nn.SyncBatchNorm.convert_sync_batchnorm): the module shells keep nn.BatchNorm2d; the
    runtimes exchange BatchNorm statistics over a process group of all ranks created here for that purpose only."""
    from ..distributed import B200DataParallel
    from ..engine.runtime import RuntimeModule
    ema_model = None
    if getattr(config, 'use_ema_model', False):
        ema_model = EmaModel(model, decay=config.ema_model_decay)
    # after the EMA copy (an eval-mode model, which never synchronizes), before the data-parallel wrapper
    if getattr(config, 'sync_bn', False) and torch.distributed.is_initialized():
        group = torch.distributed.new_group()
        for m in model.modules():
            if isinstance(m, RuntimeModule):
                m.set_bn_group(group)
    if torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
        model = B200DataParallel(model)
    return model, ema_model, None
