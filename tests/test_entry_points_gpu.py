"""The drop-in entry points end to end: each runs under torch.distributed.run on a tiny train_config.py with an in-memory
synthetic dataset for 2 epochs, writes the reference's checkpoint files and latest.pth keys, resumes to a third epoch,
and every saved model loads with strict=True into a freshly built model.  test_classification_model reproduces the acc1
that train_classification_model logged for its best checkpoint."""
import os
import re
import signal
import subprocess
import sys
import textwrap

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = 'simpleaicv_pytorch_training_examples_b200'

COMMON = f'''
import torch
from {PKG}.classification import backbones
from {PKG}.classification import losses as cls_losses


class Synthetic(torch.utils.data.Dataset):
    def __init__(self, n, size, classes, seed, labels=True):
        g = torch.Generator().manual_seed(seed)
        self.images = torch.randn(n, 3, size, size, generator=g)
        self.labels = torch.randint(0, classes, (n,), generator=g) if labels else None

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return {{'image': self.images[i]}} if self.labels is None else {{'image': self.images[i], 'label': self.labels[i]}}


def stack(batch):
    return {{k: torch.stack([b[k] for b in batch]) for k in batch[0]}}


class base:
    seed = 0
    accumulation_steps = 1
    print_interval = 1
    num_workers = 1
    use_ema_model = False
    scheduler = ('MultiStepLR', {{'warm_up_epochs': 0, 'gamma': 0.1, 'milestones': [2]}})
'''

SGD = "('SGD', {'lr': 0.01, 'momentum': 0.9, 'global_weight_decay': False, 'weight_decay': 1e-4, 'no_weight_decay_layer_name_list': []})"
ADAMW = "('AdamW', {'lr': 1e-4, 'global_weight_decay': False, 'weight_decay': 0.05, 'no_weight_decay_layer_name_list': []})"

CLASSIFICATION = f'''
class config(base):
    network = 'resnet18'
    model = backbones.resnet18(num_classes=10)
    train_criterion = cls_losses.CELoss()
    test_criterion = cls_losses.CELoss()
    train_dataset, test_dataset = Synthetic(32, 64, 10, 1), Synthetic(64, 64, 10, 2)
    train_collater = test_collater = stack
    batch_size = 8
    optimizer = {SGD}
    epochs = EPOCHS
'''

KD = f'''
from {PKG}.distillation import losses
from {PKG}.distillation.distillmodel import KDModel


class config(base):
    network = 'resnet18_kd_resnet18'
    freeze_teacher = FREEZE
    model = KDModel(teacher_type='resnet18', student_type='resnet18', freeze_teacher=freeze_teacher, num_classes=10)
    train_criterion = {{'CELoss': losses.CELoss(), 'LOSS': losses.LOSS(4.0)}}
    loss_ratio = {{'CELoss': 1.0, 'LOSS': 1.0}}
    test_criterion = losses.CELoss()
    train_dataset, test_dataset = Synthetic(32, 64, 10, 1), Synthetic(64, 64, 10, 2)
    train_collater = test_collater = stack
    batch_size = 8
    optimizer = {SGD}
    epochs = EPOCHS
'''

MAE_CFG = dict(patch_size=16, image_size=64, encoder_embedding_planes=768, encoder_block_nums=2, encoder_head_nums=12,
               decoder_embedding_planes=512, decoder_block_nums=2, decoder_head_nums=16)
MAE = f'''
from {PKG}.masked_image_modeling import losses
from {PKG}.masked_image_modeling.models import vit_mae


def patchify(batch):
    images = torch.stack([b['image'] for b in batch])
    x = images.reshape(images.shape[0], 3, 4, 16, 4, 16)
    return {{'image': images, 'label': torch.einsum('nchpwq->nhwpqc', x).reshape(images.shape[0], 16, 16 * 16 * 3)}}


class config(base):
    network = 'vit_base_patch16_224_mae_pretrain_model'
    model = vit_mae.VITMAEPretrainModel(**{MAE_CFG!r})
    train_criterion = losses.MSELoss()
    train_dataset = Synthetic(8, 64, 1, 1, labels=False)
    train_collater = patchify
    batch_size = 2
    optimizer = {ADAMW}
    epochs = EPOCHS
'''

ENCODER = f'''
from {PKG}.interactive_segmentation import distill_model
from {PKG}.interactive_segmentation.distill_losses import MSELoss

TEACHER = dict(distill_model.SAM_H_TEACHER, image_size=224, block_nums=2, global_attn_indexes=[1])
STUDENT = dict(distill_model.DINOV3_B_STUDENT, image_size=224)


class config(base):
    network = 'sam_h_encoder_distill_dinov3_vit_base_patch16_encoder'
    model = distill_model.DINOV3ImageEncoderDistillModel(teacher_params=TEACHER, student_params=STUDENT)
    freeze_teacher = True
    train_criterion = MSELoss()
    train_dataset = Synthetic(4, 224, 1, 1, labels=False)
    train_collater = stack
    batch_size = 2
    optimizer = {ADAMW}
    epochs = EPOCHS
    save_interval = 1
'''


def _write(work, name, body, **subs):
    text = COMMON + body
    for k, v in subs.items():
        text = text.replace(k, str(v))
    with open(os.path.join(work, name), 'w') as f:
        f.write(textwrap.dedent(text))


def _launch(tool, work, nproc=1, timeout=900):
    """Runs the entry point under torch.distributed.run in its own session; whatever is left of it is killed on return."""
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(nproc),
           '-m', f'{PKG}.tools.{tool}', '--work-dir', str(work)]
    # the configs are rewritten with the same size within a second: no stale bytecode for them
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE='1',
               PYTHONPATH=os.pathsep.join([ROOT] + [p for p in os.environ.get('PYTHONPATH', '').split(os.pathsep) if p]))
    proc = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                            start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=timeout)
    finally:
        try:
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
        proc.wait()
    assert proc.returncode == 0, out[-4000:]
    return out


def _load(path):
    return torch.load(path, map_location='cpu', weights_only=True)


def _train_and_resume(tool, work, body, files, latest_keys, lr, nproc=1, adamw_steps_per_epoch=None, **subs):
    """Two epochs: the checkpoint directory holds latest.pth and exactly files(latest of epoch 2).  Then the config is
    raised to three epochs: only epoch 3 runs, from the saved state, and the files of the first run stay.  `lr` is the
    config's base learning rate, which the MultiStepLR milestone at epoch 2 scales by 0.1; with AdamW, the step count of
    every parameter after epoch 3 covers all three epochs only when the optimizer state was resumed.  Returns the
    checkpoint directory, latest.pth of epochs 2 and 3 and every checkpoint file other than latest.pth."""
    _write(work, 'train_config.py', body, EPOCHS=2, **subs)
    out = _launch(tool, work, nproc)
    ckpt = os.path.join(work, 'checkpoints')
    assert re.search(r'epoch 002: train loss', out), out[-3000:]
    first = _load(os.path.join(ckpt, 'latest.pth'))
    assert set(first) == set(latest_keys) and first['epoch'] == 2
    written = files(first)
    assert sorted(os.listdir(ckpt)) == sorted(['latest.pth'] + written)
    _write(work, 'train_config.py', body, EPOCHS=3, **subs)
    out = _launch(tool, work, nproc)
    assert 'resumed from epoch 002' in out, out[-3000:]
    assert re.search(r'epoch 003: train loss', out) and not re.search(r'epoch 00[12]: train loss', out), out[-3000:]
    latest = _load(os.path.join(ckpt, 'latest.pth'))
    assert set(latest) == set(latest_keys) and latest['epoch'] == 3 and latest['time'] > first['time']
    assert abs(latest['lr'] - 0.1 * lr) <= 1e-9 * lr, (latest['lr'], lr)
    assert latest['optimizer_state_dict']['state'], 'optimizer state was not saved'
    if adamw_steps_per_epoch is not None:
        steps = {float(st['step']) for st in latest['optimizer_state_dict']['state'].values()}
        assert steps == {3. * adamw_steps_per_epoch}, steps
    now = os.listdir(ckpt)
    assert set(written) <= set(now), now
    return ckpt, first, latest, [os.path.join(ckpt, f) for f in now if f != 'latest.pth']


def _strict(module, path):
    module.load_state_dict(_load(path), strict=True)


COMMON_KEYS = {'epoch', 'time', 'lr', 'model_state_dict', 'optimizer_state_dict', 'scheduler_state_dict'}
DISTILL_KEYS = COMMON_KEYS | {'tea_best_acc1', 'tea_test_loss', 'stu_best_acc1', 'stu_test_loss'}


def _check_distill(tmp_path, loss, freeze, nproc=1):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    ckpt, first, latest, saved = _train_and_resume(
        'train_distill_classification_model', tmp_path, KD,
        lambda s: [f'teacher-epoch2-acc{s["tea_best_acc1"]:.3f}.pth', f'student-epoch2-acc{s["stu_best_acc1"]:.3f}.pth'],
        DISTILL_KEYS, 0.01, nproc, FREEZE=freeze, LOSS=loss)
    for path in saved:
        _strict(backbones.resnet18(num_classes=10), path)
    sd = latest['model_state_dict']
    assert all(k.startswith('module.teacher.') or k.startswith('module.student.') for k in sd)
    teacher_weights = [k for k in sd if k.startswith('module.teacher.') and k.endswith('.weight')]
    changed = [k for k in teacher_weights if not torch.equal(sd[k], first['model_state_dict'][k])]
    if freeze:   # a frozen teacher is not trained: its best checkpoint equals the teacher of the last epoch
        assert not changed, changed
        teacher = _load(next(p for p in saved if os.path.basename(p).startswith('teacher-')))
        assert all(torch.equal(v, sd['module.teacher.' + k]) for k, v in teacher.items())
    else:        # DML trains the teacher: epoch 3 moved every teacher weight
        assert changed == teacher_weights, sorted(set(teacher_weights) - set(changed))


def test_distill_classification_kd(tmp_path):
    _check_distill(tmp_path, 'KDLoss', True)


def test_distill_classification_dml_trains_the_teacher(tmp_path):
    _check_distill(tmp_path, 'DMLLoss', False)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
def test_distill_classification_kd_two_ranks(tmp_path):
    _check_distill(tmp_path, 'KDLoss', True, nproc=2)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
def test_distill_classification_dml_two_ranks(tmp_path):
    _check_distill(tmp_path, 'DMLLoss', False, nproc=2)


def _run_distill_ddp_check(nproc):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(nproc),
           os.path.join(ROOT, 'tests', 'distill_ddp_check.py')]
    proc = subprocess.Popen(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                            start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=900)
    finally:
        try:
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
        proc.wait()
    assert proc.returncode == 0, out[-4000:]
    assert out.count('distill ddp ok') == nproc, out[-3000:]


def test_dml_teacher_gradients_go_through_the_data_parallel_buckets():
    """N = 1: with both runtimes' sinks handed to B200DataParallel, the gradients written into its buckets equal those of
    an unwrapped copy bit for bit."""
    _run_distill_ddp_check(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
def test_dml_teacher_is_averaged_across_two_ranks():
    """N = 2: teacher and student gradients are averaged, and the parameters are bit-identical on both ranks after a step."""
    _run_distill_ddp_check(2)


def test_mae_self_supervised(tmp_path):
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling.models import vit_mae
    net = 'vit_base_patch16_224_mae_pretrain_model'
    ckpt, _, latest, saved = _train_and_resume(
        'train_mae_self_supervised_model', tmp_path, MAE,
        lambda s: [f'{net}-loss{s["best_loss"]:.3f}.pth', f'{net}-loss{s["best_loss"]:.3f}_encoder.pth'],
        COMMON_KEYS | {'best_loss', 'train_loss'}, 1e-4, adamw_steps_per_epoch=4)
    for path in saved:
        model = vit_mae.VITMAEPretrainModel(**MAE_CFG)
        _strict(model.encoder if path.endswith('_encoder.pth') else model, path)


def test_interactive_segmentation_distill_encoder(tmp_path):
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.dinov3_segment_anything.dinov3_image_encoder import \
        DINOV3ViTImageEncoder
    ckpt, _, latest, saved = _train_and_resume(
        'train_interactive_segmentation_distill_encoder_model', tmp_path, ENCODER,
        lambda s: [f'student-epoch2-loss{s["best_loss"]:.3f}.pth', 'student_model_epoch_1.pth', 'student_model_epoch_2.pth'],
        COMMON_KEYS | {'best_loss', 'train_loss'}, 1e-4, adamw_steps_per_epoch=2)
    assert os.path.join(ckpt, 'student_model_epoch_3.pth') in saved
    student = dict(distill_model.DINOV3_B_STUDENT, image_size=224)
    for path in saved:
        _strict(DINOV3ViTImageEncoder(**student), path)


def test_classification_test_tool_reproduces_the_logged_acc1(tmp_path):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    train_dir, test_dir = tmp_path / 'train', tmp_path / 'test'
    train_dir.mkdir()
    test_dir.mkdir()
    _write(train_dir, 'train_config.py', CLASSIFICATION, EPOCHS=2)
    out = _launch('train_classification_model', train_dir)
    accs = [float(a) for a in re.findall(r'epoch 00\d: train loss [-\d.naif]+, acc1 ([\d.]+)%', out)]
    assert len(accs) == 2, out[-3000:]
    best = max(accs)
    assert best > 0, 'no best checkpoint was written'
    weights = train_dir / 'checkpoints' / f'resnet18-acc{best:.3f}.pth'
    _strict(backbones.resnet18(num_classes=10), weights)
    test_config = CLASSIFICATION.replace('class config(base):', 'class config(base):\n    trained_model_path = TRAINED') + \
        '\nfrom simpleaicv_pytorch_training_examples_b200.classification.common import load_state_dict\n' \
        'load_state_dict(config.trained_model_path, config.model)\n'
    _write(test_dir, 'test_config.py', test_config, EPOCHS=2, TRAINED=repr(str(weights)))
    out = _launch('test_classification_model', test_dir)
    m = re.search(r'acc1: ([\d.]+)%, acc5: ([\d.]+)%, test_loss: ([\d.]+)', out)
    assert m, out[-3000:]
    assert m.group(1) == f'{best:.3f}', (m.group(1), best)
    assert re.search(r'model: resnet18, params: \d+', out)
    assert os.path.exists(test_dir / 'log' / 'test.info.log')
