"""ConvFormer without a GPU: the oracle (oracle/convformer.py) against the reference's recorded outputs
(tests/golden/convformer_*.ptf, written by tests/golden/make_convformer_golden.py), the product shells' state_dict
layout and seeded init, the runtime's operand list, and - when build() installed the reference into oracle/_ref - a live
comparison including the autocast(bf16) dtype flow the runtime follows."""
import glob
import importlib.util
import os

import pytest
import torch

from baseline import ref_import

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(p for p in glob.glob(os.path.join(HERE, 'golden', 'convformer_*.ptf')) if 'init' not in os.path.basename(p))
INIT = os.path.join(HERE, 'golden', 'convformer_init_c10.ptf')
ARCHS = ['convformer_s18', 'convformer_s36', 'convformer_m36', 'convformer_b36']

_spec = importlib.util.spec_from_file_location('make_convformer_golden', os.path.join(HERE, 'golden', 'make_convformer_golden.py'))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)


def test_fixtures_present():
    names = {os.path.basename(p) for p in CASES}
    assert len(names) == len(make_golden.CASES) and os.path.exists(INIT), names
    assert any(torch.load(p, weights_only=False)['drop_scales'] for p in CASES), 'no fixture exercises drop path'


@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p) for p in CASES])
def test_oracle_reproduces_reference_fixture(path):
    from oracle import convformer
    fix = torch.load(path, weights_only=False)
    torch.set_num_threads(1)
    arch, dp = fix['arch'], fix['kwargs'].get('drop_path_prob', 0.)
    sd = convformer.init_state(arch, fix['num_classes'], fix['seed'])
    assert list(sd) == fix['keys']
    assert {k: convformer.tensor_hash(v) for k, v in sd.items()} == fix['init_hash']
    scales = {k: tuple(v) for k, v in fix['drop_scales'].items()}
    if dp > 0.:
        rates = convformer.drop_path_rates(arch, dp)
        assert set(scales) == {k for k, p in rates.items() if p > 0.} and all(len(v) == 2 for v in scales.values())
    logits, loss, grads = convformer.loss_and_grads(sd, fix['x'], fix['y'], arch, drop_path_prob=dp, drop_scales=scales)
    torch.testing.assert_close(logits, fix['logits'], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(loss, fix['loss'], rtol=1e-5, atol=1e-6)
    assert set(grads) == set(fix['grad_norm'])
    for n, g in grads.items():
        assert abs(g.norm().item() - fix['grad_norm'][n]) <= 1e-5 * max(1.0, fix['grad_norm'][n]), n
        idx = make_golden.sample_index(g.numel(), n)
        torch.testing.assert_close(g.flatten()[idx], fix['grad_sample'][n], rtol=1e-5, atol=1e-6, msg=n)
    for k, v in fix['buffers'].items():
        torch.testing.assert_close(sd[k], v, rtol=1e-5, atol=1e-6)
    with torch.no_grad():
        ev = convformer.forward(sd, fix['x'], arch, training=False)
    torch.testing.assert_close(ev, fix['eval_logits'], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('arch', ARCHS)
def test_shells_match_reference_layout_and_init(arch):
    from oracle import convformer
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    ref = torch.load(INIT, weights_only=False)
    want = ref['archs'][arch]
    torch.manual_seed(ref['seed'])
    sd = backbones.__dict__[arch](num_classes=ref['num_classes']).state_dict()
    assert list(sd) == want['keys']
    assert {k: tuple(v.shape) for k, v in sd.items()} == want['shapes']
    assert {k: convformer.tensor_hash(v) for k, v in sd.items()} == want['hash']
    osd = convformer.init_state(arch, ref['num_classes'], ref['seed'])
    assert {k: convformer.tensor_hash(v) for k, v in osd.items()} == want['hash']


def test_constructor_surface():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    m = backbones.__dict__['convformer_s18'](inplanes=3, dropout_prob=0., drop_path_prob=0.2, num_classes=7, use_gradient_checkpoint=True)
    assert m.use_gradient_checkpoint and m.head.out_features == 7
    assert m.stages[0][0].drop_path.__class__.__name__ == 'Identity' and m.stages[3][2].drop_path.drop_path_prob == pytest.approx(0.2)
    with pytest.raises(NotImplementedError):
        backbones.convformer_s18(dropout_prob=0.1)
    with pytest.raises(RuntimeError, match='GPU'):
        backbones.convformer_s18(num_classes=10)(torch.zeros(1, 3, 64, 64))


@pytest.mark.parametrize('arch', ['convformer_s18', 'convformer_m36'])
def test_runtime_lists_every_gemm_weight_once_in_launch_order(arch):
    import test_operands_cpu
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.engine.operands import CONV, ROWS, STEM
    torch.manual_seed(0)
    model = backbones.__dict__[arch](num_classes=10)
    ops = model._runtime().operands()
    names = {id(p): n for n, p in model.named_parameters()}
    listed = [names.get(id(op.param)) for op in ops]
    assert None not in listed and len(set(listed)) == len(listed)
    assert set(listed) == test_operands_cpu._gemm_weights(model)
    assert all(op.w is None for op in ops), 'building the runtime allocated an operand copy'
    want = []
    for i, stage in enumerate(model.stages):
        want.append((f'downsample_layers.{i}.conv.weight', STEM if i == 0 else CONV))
        for j in range(len(stage)):
            b = f'stages.{i}.{j}'
            want += [(f'{b}.token_mixer.pwconv1.weight', ROWS), (f'{b}.token_mixer.pwconv2.weight', ROWS),
                     (f'{b}.mlp.fc1.weight', ROWS), (f'{b}.mlp.fc2.weight', ROWS)]
    want.append(('head.weight', ROWS))
    assert [(names[id(op.param)], op.layout) for op in ops] == want


needs_ref = pytest.mark.skipif(not ref_import.available(), reason='reference not installed (oracle/build_ref.py)')


@needs_ref
@pytest.mark.parametrize('dp', [0., 0.3])
def test_oracle_matches_live_reference(dp):
    """oracle/convformer.py vs SimpleAICV/classification/backbones/convformer.py (seeded init, logits, every gradient),
    with the reference's own drop-path draws replayed."""
    from oracle import convformer
    torch.manual_seed(3)
    ref = ref_import.backbones().convformer_s18(num_classes=10, drop_path_prob=dp)
    sd = convformer.init_state('convformer_s18', 10, 3)
    rs = ref.state_dict()
    assert list(rs) == list(sd) and all(torch.equal(rs[k], sd[k]) for k in rs)
    scales = make_golden.record_drop_scales(ref)
    g = torch.Generator().manual_seed(12)
    x, y = torch.randn(3, 3, 64, 64, generator=g), torch.randint(0, 10, (3,), generator=g)
    ref.train()
    out = ref(x)
    torch.nn.functional.cross_entropy(out, y).backward()
    lo, _, gr = convformer.loss_and_grads(sd, x, y, 'convformer_s18', drop_path_prob=dp,
                                          drop_scales={k: tuple(v) for k, v in scales.items() if v})
    torch.testing.assert_close(lo, out.detach(), rtol=1e-5, atol=1e-5)
    for n, p in ref.named_parameters():
        torch.testing.assert_close(gr[n], p.grad, rtol=1e-4, atol=1e-6, msg=n)
    for k in rs:
        if 'running' in k:
            torch.testing.assert_close(sd[k], ref.state_dict()[k], rtol=1e-5, atol=1e-6, msg=k)


@needs_ref
def test_reference_dtype_flow_under_autocast():
    """The dtype flow the runtime and the oracle's emulate_bf16 follow, read off the live reference under CPU
    autocast(bf16): downsampling outputs bf16; in training the stream turns fp32 at the first block that applies a drop
    path (fp32 mask, convformer.py:131-137) - stage 1 block 0 has p = 0 and stays bf16 -; in eval mode, or with
    drop_path_prob = 0, it stays bf16; the pooled features have the stream's dtype and the logits are bf16."""
    torch.manual_seed(0)

    def run(dp, training):
        model = ref_import.backbones().convformer_s18(num_classes=10, drop_path_prob=dp).train(training)
        seen = {}
        for i, d in enumerate(model.downsample_layers):
            d.register_forward_hook(lambda m, a, o, i=i: seen.__setitem__(f'down{i}', o.dtype))
        for i, st in enumerate(model.stages):
            for j, b in enumerate(st):
                b.register_forward_hook(lambda m, a, o, k=f'{i}.{j}': seen.__setitem__(k, o.dtype))
        model.avgpool.register_forward_hook(lambda m, a, o: seen.__setitem__('pool', o.dtype))
        with torch.autocast('cpu', dtype=torch.bfloat16), torch.no_grad():
            seen['logits'] = model(torch.randn(2, 3, 64, 64)).dtype
        return seen

    bf, f32 = torch.bfloat16, torch.float32
    tr = run(0.2, True)
    assert all(tr[f'down{i}'] == bf for i in range(4)) and tr['logits'] == bf
    assert tr['0.0'] == bf and tr['0.1'] == f32 and tr['0.2'] == f32
    assert all(tr[f'{i}.{j}'] == f32 for i, n in ((1, 3), (2, 9), (3, 3)) for j in range(n)) and tr['pool'] == f32
    for seen in (run(0.2, False), run(0., True)):
        assert all(v == bf for v in seen.values()), seen
