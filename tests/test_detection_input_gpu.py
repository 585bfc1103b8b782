"""DETR and SAM-encoder inputs on the uint8 edge, device side: CudaPrefetcher's batches from ResizePadBatch records equal
the committed oracle fixture and the oracle at 1024^2 bit for bit (image and DETR mask, mixed sizes, translations, SAM
flips); train_detection, train_distill_sam_encoder and test_detection fed by the uint8 path give the losses, parameters
(DETR's within its own run-to-run spread) and decoded boxes of the fp32 path fed the oracle's batches."""
import importlib.util
import logging
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_detection_input', os.path.join(HERE, 'golden', 'make_detection_input_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)
SAM_NORM = ((123.675, 116.28, 103.53), (58.395, 57.12, 57.375))


def _prefetch(batches):
    from simpleaicv_pytorch_training_examples_b200.tools.utils import CudaPrefetcher
    return [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in b.items()} for b in CudaPrefetcher(batches)]


def _fixture_batch(z, kind, seed):
    from simpleaicv_pytorch_training_examples_b200.detection.common import ResizePadBatch
    p = f'{kind}{seed}_'
    norm = (None, None) if kind == 'detr' else SAM_NORM
    return ResizePadBatch(torch.from_numpy(z[p + 'data']), torch.from_numpy(z[p + 'offsets']), torch.from_numpy(z[p + 'geom']),
                          torch.from_numpy(z[p + 'shift']), mk.RESIZE, *norm, with_mask=kind == 'detr')


def test_prefetched_batches_equal_the_fixture():
    z = np.load(mk.FIXTURE)
    cases = [('detr', s) for s, _ in mk.DETR_BATCHES] + [('sam', s) for s, _ in mk.SAM_BATCHES]
    got = _prefetch([{'resize_pad': _fixture_batch(z, k, s), 'tag': f'{k}{s}_'} for k, s in cases])
    for (kind, seed), b in zip(cases, got):
        p = b['tag']
        assert torch.equal(b['image'].cpu().view(torch.int32), torch.from_numpy(z[p + 'oracle_image']).view(torch.int32)), p
        if kind == 'detr':
            assert torch.equal(b['mask'].cpu(), torch.from_numpy(z[p + 'oracle_mask'])), p
        else:
            assert 'mask' not in b


@pytest.mark.parametrize('kind', ['detr', 'sam'])
def test_1024_batches_equal_the_oracle(kind):
    from simpleaicv_pytorch_training_examples_b200.detection.common import ResizePadBatch
    rng = np.random.RandomState(5)
    shapes = [(480, 640), (640, 427), (1024, 768), (1500, 2250), (333, 500), (20, 1024)]
    srcs = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in shapes]
    geom, shift = [], []
    for i, (h, w) in enumerate(shapes):
        f = (1024 if kind == 'sam' else (800, 1024)[i % 2]) / max(h, w)
        tr = int(kind == 'detr' and i % 3 != 2)
        geom.append([h, w, int(round(h * f)), int(round(w * f)), int(kind == 'sam' and i % 2 == 0), tr])
        shift.append(rng.uniform(-40, 40, size=2) if tr else np.zeros(2))
    sizes = [s.size for s in srcs]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    rp = ResizePadBatch(torch.from_numpy(np.concatenate([s.reshape(-1) for s in srcs])), torch.from_numpy(offsets),
                        torch.tensor(geom, dtype=torch.int32), torch.tensor(np.array(shift), dtype=torch.float64), 1024,
                        *(SAM_NORM if kind == 'sam' else (None, None)), with_mask=kind == 'detr')
    (got,) = _prefetch([{'resize_pad': rp}])
    image, mask = mk.oracle_batch(rp)
    assert torch.equal(got['image'].cpu().view(torch.int32), torch.from_numpy(image).view(torch.int32))
    if kind == 'detr':
        assert torch.equal(got['mask'].cpu(), torch.from_numpy(mask))


def test_bad_records_are_rejected_before_any_launch():
    from simpleaicv_pytorch_training_examples_b200 import ops
    from simpleaicv_pytorch_training_examples_b200.detection.common import ResizePadBatch
    src = torch.zeros(10 * 10 * 3, dtype=torch.uint8, device='cuda')
    for geom, shift in [([10, 11, 10, 10, 0, 0], [0, 0]), ([10, 10, 65, 10, 0, 0], [0, 0]), ([10, 10, 10, 10, 2, 0], [0, 0]),
                        ([10, 10, 10, 10, 0, 1], [float('nan'), 0]), ([10, 10, 0, 10, 0, 0], [0, 0])]:
        rp = ResizePadBatch(None, torch.zeros(1, dtype=torch.int64), torch.tensor([geom], dtype=torch.int32),
                            torch.tensor([shift], dtype=torch.float64), 64)
        with pytest.raises(RuntimeError, match='saicv_u8_resize_pad'):
            ops.u8_resize_pad(src, rp)


def _detr_batches(n_batches, resize):
    """Uint8DETRDetectionCollater batches of the DETR chain at ``resize``, and the same batches with the oracle's fp32
    'image' and 'mask' in place of the record (what the reference's collater gives, up to cv2's IPP)."""
    from simpleaicv_pytorch_training_examples_b200.detection import common as udet
    u8, f32 = [], []
    for seed in range(n_batches):
        samples = mk.detr_samples(10 + seed, [(96, 128), (128, 90), (60, 160), (140, 100)])
        b, _ = mk.run(samples, mk.detr_chain(udet, resize, 'Uint8'),
                      udet.Uint8DETRDetectionCollater(resize=resize, resize_type='yolo_style', max_annots_num=8,
                                                      pin_memory=False), seed)
        image, mask = mk.oracle_batch(b['resize_pad'])
        u8.append(b)
        f32.append(dict({k: v for k, v in b.items() if k != 'resize_pad'}, image=torch.from_numpy(image),
                        mask=torch.from_numpy(mask)))
    return u8, f32


class _Sched:
    current_lr = 1e-4

    def step(self, optimizer, epoch):
        pass


def _train(model_fn, fn, batches, cfg, criterion):
    from simpleaicv_pytorch_training_examples_b200 import optim

    class Loader(list):
        dataset = list(range(len(batches) * 4))

    torch.manual_seed(0)
    model = model_fn()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = optim.FusedAdamW([{'params': params, 'weight_decay': 0.}], lr=1e-4)
    avg = fn(Loader(batches), model, criterion, opt, _Sched(), 1, logging.getLogger('t'), cfg)
    torch.cuda.synchronize()
    return avg, {n: p.detach().cpu().clone() for n, p in model.named_parameters()}


def test_train_detection_uint8_equals_fp32_oracle_batches():
    from simpleaicv_pytorch_training_examples_b200.detection import losses, models
    from simpleaicv_pytorch_training_examples_b200.tools import scripts

    class Cfg:
        network, accumulation_steps, batch_size, print_interval, local_rank = 'resnet18_detr', 1, 4, 1, 0

    def model_fn():
        m = models.resnet18_detr(num_classes=80).cuda()
        m.transformer.dropout_prob = 0.0
        return m

    u8, f32 = _detr_batches(1, 160)
    # the model sees the same bits on both paths
    for x, y in zip(_prefetch(u8), _prefetch(f32)):
        for k in ('image', 'mask', 'annots', 'scaled_annots'):
            assert torch.equal(x[k].cpu(), y[k].cpu()), k
    crit = losses.DETRLoss(num_classes=80)
    torch.manual_seed(0)
    p0 = {n: p.detach().cpu().clone() for n, p in model_fn().named_parameters()}
    a, pa = _train(model_fn, scripts.train_detection, u8, Cfg, crit)
    b, pb = _train(model_fn, scripts.train_detection, f32, Cfg, crit)
    assert a == b and a > 0
    # DETR-R18's weight gradients are not bit-reproducible run to run (split reductions), so the updated parameters are
    # held to a small fraction of the step itself
    for n in pa:
        step = (pb[n] - p0[n]).abs().max()
        assert (pa[n] - pb[n]).abs().max() <= 1e-2 * step, n


def test_test_detection_uint8_gives_the_decoded_boxes_of_fp32_oracle_batches(monkeypatch):
    from simpleaicv_pytorch_training_examples_b200.detection import decode, losses, models
    from simpleaicv_pytorch_training_examples_b200.tools import scripts
    u8, f32 = _detr_batches(2, 160)
    torch.manual_seed(0)
    model = models.resnet18_detr(num_classes=80).cuda()
    seen = []
    monkeypatch.setattr(scripts, '_evaluate_detections', lambda index, arrays, config: seen.append(arrays['decoded']) or {})

    class Cfg:
        network, eval_type, batch_size, gpus_num = 'resnet18_detr', 'VOC', 4, 1

    class Loader(list):
        sampler = list(range(8))

    dec = decode.DETRDecoder(num_classes=80, max_object_num=100, min_score_threshold=0.0, topn=100, nms_type=None,
                             nms_threshold=0.5)
    ra = scripts.test_detection(Loader(u8), model, losses.DETRLoss(num_classes=80), dec, Cfg)
    rb = scripts.test_detection(Loader(f32), model, losses.DETRLoss(num_classes=80), dec, Cfg)
    assert ra['test_loss'] == rb['test_loss']
    assert len(seen) == 2 and seen[0].shape == seen[1].shape and np.array_equal(seen[0], seen[1])


def test_train_distill_sam_encoder_uint8_equals_fp32_oracle_batches():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import common as usam
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.distill_losses import MSELoss
    from simpleaicv_pytorch_training_examples_b200.tools import interactive_segmentation_scripts as iss
    u8, f32 = [], []
    for seed in range(2):
        samples = mk.sam_samples(20 + seed, [(240, 320), (320, 200), (150, 90)])
        b, _ = mk.run(samples, mk.sam_chain(usam, 320, 'Uint8'), usam.Uint8SAMBatchCollater(resize=320, pin_memory=False), seed)
        image, _ = mk.oracle_batch(b['resize_pad'])
        u8.append(b)
        f32.append(dict({k: v for k, v in b.items() if k != 'resize_pad'}, image=torch.from_numpy(image)))

    class Cfg:
        accumulation_steps, batch_size, print_interval, local_rank, freeze_teacher = 1, 3, 1, 0, True

    def model_fn():
        tea = dict(distill_model.SAM_H_TEACHER, image_size=320, block_nums=2, global_attn_indexes=[1])
        stu = dict(distill_model.DINOV3_B_STUDENT, image_size=320)
        return distill_model.DINOV3ImageEncoderDistillModel(teacher_params=tea, student_params=stu).cuda()

    a, pa = _train(model_fn, iss.train_distill_sam_encoder, u8, Cfg, MSELoss())
    b, pb = _train(model_fn, iss.train_distill_sam_encoder, f32, Cfg, MSELoss())
    assert a == b and a > 0
    for n in pa:
        assert torch.equal(pa[n], pb[n]), n
