"""Host-side helpers of the classification hot path with the reference's names
(SimpleAICV/classification/common.py:668-685 AverageMeter, :688-709 AccMeter, :843-881 get_amp_type) and the
input-pipeline edge of SURVEY.md 8 f3: ``Uint8ClassificationCollater`` + ``DeviceNormalize`` move the batch over PCIe as
uint8 pixels and normalise on the device.  The per-sample transforms / datasets stay CPU data code (SURVEY.md section 2)."""
import numpy as np
import torch


def load_state_dict(saved_model_path, model, excluded_layer_name=()):
    """classification/common.py:758-800 of the reference: loads the entries of a saved ``state_dict`` file whose name and
    shape match ``model`` (and whose name contains none of ``excluded_layer_name``); an empty path is a no-op."""
    if not saved_model_path:
        return
    saved = torch.load(saved_model_path, map_location=torch.device('cpu'), weights_only=True)
    own = model.state_dict()
    keep = {n: w for n, w in saved.items()
            if n in own and w.shape == own[n].shape and not any(e in n for e in excluded_layer_name)}
    skipped = [n for n in saved if n not in keep]
    if skipped:
        print(f'not loaded: {len(skipped)} of {len(saved)} saved tensors (name / shape mismatch or excluded)')
    model.load_state_dict(keep, strict=False)


class Uint8ClassificationCollater:
    """Counterpart of ClassificationCollater (common.py:645-665) for samples whose 'image' is still the decoder's uint8
    [H, W, 3] array (i.e. the transform list ends BEFORE TorchMeanStdNormalize / Normalize): stacks into ONE pinned uint8
    [B, H, W, 3] tensor (a quarter of the fp32 batch's bytes on the host link) and int64 labels.  ``DeviceNormalize`` (or
    tools.utils.CudaPrefetcher(normalize=...)) finishes the reference's arithmetic on the GPU."""

    def __init__(self, pin_memory=True):
        self.pin_memory = pin_memory

    def __call__(self, data):
        images = np.stack([np.ascontiguousarray(s['image']) for s in data])
        assert images.dtype == np.uint8 and images.ndim == 4 and images.shape[3] == 3, 'expects uint8 [H, W, 3] images'
        labels = torch.from_numpy(np.array([s['label'] for s in data]).astype(np.float32)).long()
        images = torch.from_numpy(images)
        if self.pin_memory and torch.cuda.is_available():
            images, labels = images.pin_memory(), labels.pin_memory()
        return {'image': images, 'label': labels}


class DeviceNormalize:
    """(x / 255 - mean) / std and NHWC -> NCHW on the device (csrc/capi_input.cu): TorchMeanStdNormalize
    (common.py:228-248; mean / std given) or Normalize (:190-206; mean 0, std 1 -> x / 255) followed by the collater's
    permute, bit-identical to the host pipeline.  Raises on CPU tensors: there is no host fallback."""

    def __init__(self, mean=(0., 0., 0.), std=(1., 1., 1.)):
        self.mean, self.std = tuple(float(v) for v in mean), tuple(float(v) for v in std)

    def __call__(self, images_u8, out=None):
        from .. import ops
        if not images_u8.is_cuda:
            raise RuntimeError('DeviceNormalize runs on the GPU (uint8 [B, H, W, 3] device tensor expected)')
        return ops.u8_normalize(images_u8, self.mean, self.std, out=out)


class AverageMeter:
    """Running average (sum of val*n over count)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.val, self.avg, self.sum, self.count = 0, 0, 0, 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


class AccMeter:
    """Accumulates top-1 / top-5 correct counts; ``compute()`` fills ``acc1`` / ``acc5`` as fractions."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.acc1_correct_num = 0
        self.acc5_correct_num = 0
        self.sample_num = 0
        self.acc1 = 0
        self.acc5 = 0

    def update(self, acc1_correct_num, acc5_correct_num, sample_num):
        self.acc1_correct_num += acc1_correct_num
        self.acc5_correct_num += acc5_correct_num
        self.sample_num += sample_num

    def compute(self):
        self.acc1 = float(self.acc1_correct_num) / self.sample_num if self.sample_num != 0 else 0
        self.acc5 = float(self.acc5_correct_num) / self.sample_num if self.sample_num != 0 else 0


class SemanticSoftmaxMeter:
    """common.py:712-757 of the reference: accuracy over the semantic tree's levels, counting every (row, level) pair that
    has a label.  compute_per_batch runs one kernel (csrc/capi_loss.cu: first argmax per level, torch.argmax's NaN rule)
    on the SemanticOutputs' full logits and returns (correct, valid) as int64 device scalars: the reference's
    ``result = sum_l mean_valid(correct) * n_valid`` is that integer.  The counts stay on the device until compute()."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.acc1 = 0
        self.sum = 0
        self.count = 0

    def compute_per_batch(self, semantic_outputs, semantic_labels):
        from .. import ops
        from .semantic import SemanticOutputs
        if not isinstance(semantic_outputs, SemanticOutputs):
            raise TypeError('SemanticSoftmaxMeter takes the SemanticOutputs of SemanticTree.convert_outputs_to_semantic_outputs')
        logits = semantic_outputs.logits
        if not logits.is_cuda:
            raise RuntimeError('SemanticSoftmaxMeter runs on H100 kernels only; move the logits to the GPU')
        if logits.dtype not in (torch.float32, torch.bfloat16):
            logits = logits.float()
        t = semantic_outputs.tree.tables(logits.device)
        counts = ops.semantic_accuracy(logits.contiguous(), semantic_labels.long().contiguous(), t.level_cols, t.level_off)
        total = counts.sum(dim=0, dtype=torch.int64)
        return total[0], total[1]

    def update_per_batch(self, result, num_valids_total):
        self.sum += result
        self.count += num_valids_total

    def compute(self):
        count = int(self.count)
        self.acc1 = float(self.sum) / count if count != 0 else 0


def get_amp_type(model):
    """The autocast dtype the reference's loop would select for the device ``model`` lives on.

    Same decision procedure as the reference (compute capability >= 8, torch >= 1.10, CUDA >= 11, device
    name in a whitelist) with 'B200' (and 'B300' / 'GB200') added to the whitelist: the unmodified list
    lacks Blackwell parts, so the reference falls back to fp16 + GradScaler on a B200 (SURVEY.md 0.5).
    The kernels of this package always compute in bf16 with fp32 accumulation; the value is what
    ``train_config`` / the loops report and what a torch-side tail (criterion) may autocast to."""
    device = next(model.parameters()).device
    if device.type != 'cuda':
        return torch.bfloat16
    properties = torch.cuda.get_device_properties(device)
    ok = properties.major >= 8
    ver = tuple(int(v) for v in torch.__version__.split('+')[0].split('.')[:2])
    ok = ok and ver >= (1, 10)
    if torch.version.cuda and float(torch.version.cuda.split('.')[0]) < 11:
        ok = False
    name = torch.cuda.get_device_name(device)
    whitelist = ['RTX PRO 6000', 'H20', 'L20', 'L40', '4090', '5090', 'A100', 'A800', 'H100', 'H800',
                 'B200', 'B300', 'GB200']
    ok = ok and any(n in name for n in whitelist)
    return torch.bfloat16 if ok else torch.float16
