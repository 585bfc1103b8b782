"""SemanticSoftmaxLoss / SemanticSoftmaxMeter on the H100 kernels (csrc/capi_loss.cu) against the float64 oracle
(oracle/semantic_softmax.py) and the reference fixture (tests/golden/make_semantic_softmax_golden.py), and the ImageNet-21K
training step of a ResNet-18 with 10 450 classes: reproducible, capturable, head gradients against the oracle."""
import importlib.util
import os

import pytest
import torch

from oracle import semantic_softmax as osem

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_semantic', os.path.join(HERE, 'golden', 'make_semantic_softmax_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)
NC = sum(mk.LARGE_DEPTH_COUNTS)
ADAMW = ('AdamW', {'lr': 2e-3, 'global_weight_decay': False, 'weight_decay': 1e-4, 'no_weight_decay_layer_name_list': []})


class _TreeData:
    def __init__(self, class_tree_list, hierarchy_indices_list=None, normalization_factor_list=None):
        self.class_tree_list = class_tree_list
        if hierarchy_indices_list is None:
            hierarchy_indices_list, normalization_factor_list = osem.tree_levels(class_tree_list)
        self.hierarchy_indices_list, self.normalization_factor_list = hierarchy_indices_list, normalization_factor_list


@pytest.fixture(scope='module')
def big():
    from simpleaicv_pytorch_training_examples_b200.classification.semantic import SemanticTree
    data = _TreeData(mk.make_tree(mk.LARGE_DEPTH_COUNTS, seed=0)['class_tree_list'])
    return data, SemanticTree(data)


def _labels(data, b, seed):
    """Random classes with a shallow class and a maximum-depth class among them."""
    g = torch.Generator().manual_seed(seed)
    depth = torch.tensor([len(c) - 1 for c in data.class_tree_list])
    y = torch.randint(0, len(depth), (b,), generator=g)
    y[0] = int(torch.nonzero(depth == 2)[0])
    if b > 1:
        y[1] = int(torch.nonzero(depth == int(depth.max()))[0])
    return y


@pytest.mark.parametrize('smoothing', [0.2, 0.])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('B', [1, 7, 256])
def test_loss_and_gradient_match_float64_oracle(big, B, dtype, smoothing):
    from simpleaicv_pytorch_training_examples_b200 import ops
    data, tree = big
    t = tree.tables('cuda')
    g = torch.Generator().manual_seed(B * 10 + int(smoothing * 10))
    x = (torch.randn(B, NC, generator=g) * 3).to(dtype)
    y = _labels(data, B, B)
    sem = tree.convert_single_labels_to_semantic_labels(y.cuda())
    loss, lse = ops.semantic_softmax_fwd(x.cuda(), sem, t.level_cols, t.level_off, t.factors, smoothing)
    dx = ops.semantic_softmax_bwd(x.cuda(), sem, t.col_level, t.level_cols, t.level_off, t.factors, lse,
                                  torch.ones((), device='cuda'), smoothing).cpu()
    factors = data.normalization_factor_list.double()
    ref_loss, ref_dx = osem.loss_and_grad(x.double(), sem.cpu(), data.hierarchy_indices_list, factors, smoothing)
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)), (float(loss), float(ref_loss))
    col_level = t.col_level.long().cpu()
    f_col = torch.where(col_level >= 0, factors.float()[col_level.clamp(min=0)], torch.zeros(()))
    err = (dx.double() - ref_dx).abs()
    bound = 1e-6 * f_col.double() / B + 1e-5 * ref_dx.abs()
    assert (err <= bound).all(), f'{int((err > bound).sum())} elements off, worst excess {float((err - bound).max()):.3g}'
    assert (dx[:, col_level < 0] == 0).all()                      # columns of no level: exactly 0
    sem_c = sem.cpu()
    for lv in range(sem_c.shape[1]):
        rows = sem_c[:, lv] < 0
        if rows.any():
            assert (dx[rows][:, col_level == lv] == 0).all()      # invalid (row, level) pairs: exactly 0
    if dtype == torch.float32:   # the public loss runs the same kernels: bit-identical to the direct calls
        from simpleaicv_pytorch_training_examples_b200.classification.losses import SemanticSoftmaxLoss
        xc = x.cuda().requires_grad_(True)
        out = SemanticSoftmaxLoss(data.normalization_factor_list, smoothing)(tree.convert_outputs_to_semantic_outputs(xc), sem)
        out.backward()
        assert torch.equal(out.detach(), loss) and torch.equal(xc.grad.cpu(), dx)


def test_fixture_reproduces_through_public_loss_and_meter():
    from simpleaicv_pytorch_training_examples_b200.classification.common import SemanticSoftmaxMeter
    from simpleaicv_pytorch_training_examples_b200.classification.losses import SemanticSoftmaxLoss
    from simpleaicv_pytorch_training_examples_b200.classification.semantic import SemanticTree
    fix = torch.load(os.path.join(HERE, 'golden', 'semantic_softmax_c316_b24.pts'), weights_only=False)
    tree = SemanticTree(_TreeData(fix['tree']['class_tree_list'], fix['hierarchy_indices_list'], fix['normalization_factor_list']))
    sem = tree.convert_single_labels_to_semantic_labels(fix['labels'].cuda())
    assert torch.equal(sem.cpu(), fix['semantic_labels'])
    for s in (0.2, 0.):
        crit = SemanticSoftmaxLoss(fix['normalization_factor_list'], smoothing=s).cuda()
        x = fix['logits'].cuda().requires_grad_(True)
        loss = crit(tree.convert_outputs_to_semantic_outputs(x), sem)
        loss.backward()
        torch.testing.assert_close(loss.detach().cpu(), fix[f'loss_s{s}'], rtol=1e-5, atol=0)
        torch.testing.assert_close(x.grad.cpu(), fix[f'grad_s{s}'], rtol=1e-5, atol=1e-7)
    meter = SemanticSoftmaxMeter()
    result, valid = meter.compute_per_batch(tree.convert_outputs_to_semantic_outputs(fix['logits'].cuda()), sem)
    assert int(result) == round(float(fix['meter_result'])) and int(valid) == int(fix['meter_valid'])
    meter.update_per_batch(result, valid)
    meter.update_per_batch(result, valid)
    meter.compute()
    assert meter.acc1 == int(result) / int(valid)
    # ties and a NaN row follow torch.argmax (first maximum; NaN is the maximum)
    x = fix['logits'].clone()
    hier = fix['hierarchy_indices_list']
    x[8, hier[1]] = 1.0                                   # a level where every column ties
    x[9, hier[2][5]] = float('nan')
    x[9, hier[2][7]] = float('nan')
    x[10, hier[3]] = float('-inf')
    xc = x.cuda()
    out = tree.convert_outputs_to_semantic_outputs(xc)
    got = SemanticSoftmaxMeter().compute_per_batch(out, sem)
    ref = osem.accuracy_counts(xc, sem, [ix.cuda() for ix in hier])
    assert (int(got[0]), int(got[1])) == (int(ref[:, 0].sum()), int(ref[:, 1].sum()))
    from simpleaicv_pytorch_training_examples_b200 import ops
    t = tree.tables('cuda')
    for dtype in (torch.float32, torch.bfloat16):
        counts = ops.semantic_accuracy(xc.to(dtype), sem, t.level_cols, t.level_off).long().cpu()
        assert torch.equal(counts, osem.accuracy_counts(xc.to(dtype), sem, [ix.cuda() for ix in hier]))


def test_no_host_sync_in_conversion_loss_and_backward(big):
    from simpleaicv_pytorch_training_examples_b200.classification.losses import SemanticSoftmaxLoss
    data, tree = big
    crit = SemanticSoftmaxLoss(data.normalization_factor_list, 0.2)
    y = _labels(data, 16, 3).cuda()
    x = torch.randn(16, NC, device='cuda', requires_grad=True)

    def step():
        loss = crit(tree.convert_outputs_to_semantic_outputs(x), tree.convert_single_labels_to_semantic_labels(y))
        loss.backward()
        return loss

    step()                                   # the tables and the factors reach the device once
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _model_and_opt(seed=0):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils

    class Cfg:
        optimizer = ADAMW
    torch.manual_seed(seed)
    m = backbones.resnet18(num_classes=NC).cuda().train()
    opt = tutils.build_optimizer(Cfg, m)[0]
    assert type(opt).__name__ == 'FusedAdamW'
    return m, opt


def _batch(data):
    g = torch.Generator().manual_seed(7)
    return torch.randn(8, 3, 64, 64, generator=g).cuda(), _labels(data, 8, 7).cuda()


def _criterion(data, tree):
    from simpleaicv_pytorch_training_examples_b200.classification.losses import SemanticSoftmaxLoss
    crit = SemanticSoftmaxLoss(data.normalization_factor_list, 0.2)
    return lambda logits, y: crit(tree.convert_outputs_to_semantic_outputs(logits), tree.convert_single_labels_to_semantic_labels(y))


def test_model_steps_are_bit_reproducible_and_capturable(big):
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    data, tree = big
    x, y = _batch(data)
    crit = _criterion(data, tree)
    runs = []
    for _ in range(2):
        m, opt = _model_and_opt()
        losses = []
        for _ in range(3):
            loss = crit(m(x), y)
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.detach().clone())
        runs.append((m, losses))
    torch.cuda.synchronize()
    (m1, l1), (m2, l2) = runs
    assert all(torch.equal(a, b) for a, b in zip(l1, l2))
    for (n, p), q in zip(m1.named_parameters(), m2.parameters()):
        assert torch.equal(p, q), n
    del runs, m1, m2
    me, oe = _model_and_opt()
    mg, og = _model_and_opt()
    graphed = GraphedTrainStep(mg, crit, og, x, y, warmup=2)         # two eager warm-up steps, then the capture
    for _ in range(2):
        loss = crit(me(x), y)
        loss.backward()
        oe.step()
        oe.zero_grad()
    for _ in range(2):
        lg = graphed(x, y).clone()
        loss = crit(me(x), y)
        loss.backward()
        oe.step()
        oe.zero_grad()
        assert torch.equal(lg, loss.detach())
    torch.cuda.synchronize()
    for (n, p), q in zip(me.named_parameters(), mg.parameters()):
        assert torch.equal(p, q), n


def test_head_gradients_match_oracle_fed_the_same_dlogits(big):
    """Teacher-forced head (as tests/test_resnet_gpu.py's stage-wise parity): the oracle's last feature map through the
    runtime's head, the kernel's logit gradient (itself checked against the float64 oracle) through both heads; the fc
    gradients agree to the relative L2 that test uses for parameters (3e-2)."""
    from oracle import convnets
    from simpleaicv_pytorch_training_examples_b200 import ops
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    data, tree = big
    x, y = _batch(data)
    sd = convnets.init_state('resnet18', NC, 0)
    for n in convnets.param_names(sd):
        sd[n].requires_grad_(True)
    trace = {}
    logits = convnets.forward(sd, x.cpu(), 'resnet18', training=True, emulate_bf16=True, trace=trace)
    t = tree.tables('cuda')
    sem = tree.convert_single_labels_to_semantic_labels(y)
    lg = logits.detach().float().cuda().contiguous()
    _, lse = ops.semantic_softmax_fwd(lg, sem, t.level_cols, t.level_off, t.factors, 0.2)
    dl = ops.semantic_softmax_bwd(lg, sem, t.col_level, t.level_cols, t.level_off, t.factors, lse, torch.ones((), device='cuda'), 0.2)
    _, ref_dl = osem.loss_and_grad(logits.detach(), sem.cpu(), data.hierarchy_indices_list, data.normalization_factor_list.double(), 0.2)
    assert ((dl.cpu().double() - ref_dl).norm() / ref_dl.norm()).item() < 1e-5
    logits.backward(dl.cpu())
    torch.manual_seed(0)
    model = backbones.resnet18(num_classes=NC).cuda().train()
    rt = model._runtime()
    rt.prep()
    tape = {}
    last = trace[f'block{len(rt.blocks) - 1}_out'].detach().permute(0, 2, 3, 1).contiguous()
    rt.head_forward(last.to(torch.bfloat16).cuda(), tape)
    rt.head_backward(dl, tape)
    torch.cuda.synchronize()
    for name, p in (('fc.weight', model.fc.weight), ('fc.bias', model.fc.bias)):
        ref = sd[name].grad
        rel = ((p.grad.float().cpu() - ref).norm() / ref.norm()).item()
        assert rel <= 3e-2, (name, rel)
