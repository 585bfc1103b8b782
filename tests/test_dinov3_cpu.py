"""DINOv3 without a GPU: the oracle (oracle/dinov3.py) against the reference's recorded outputs (tests/golden/dinov3_*.ptf,
written by tests/golden/make_dinov3_golden.py), the shells' state_dict layout and seeded init against the reference, the
RoPE rescale draw, the refusals, and the runtime's operand list."""
import glob
import importlib.util
import os

import pytest
import torch

from baseline import ref_import

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(glob.glob(os.path.join(HERE, 'golden', 'dinov3_*.ptf')))
_spec = importlib.util.spec_from_file_location('make_dinov3_golden', os.path.join(HERE, 'golden', 'make_dinov3_golden.py'))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)
BUILT = ['dinov3_vit_small_patch16_backbone', 'dinov3_vit_small_plus_patch16_backbone', 'dinov3_vit_base_patch16_backbone',
         'dinov3_vit_large_patch16_backbone', 'dinov3_vit_large_plus_patch16_backbone', 'dinov3_vit_huge_plus_patch16_backbone']
needs_ref = pytest.mark.skipif(not ref_import.available(), reason='reference not installed (oracle/build_ref.py)')


def oracle_state(fix):
    from oracle import dinov3 as od
    if fix['kind'] == 'encoder':
        c, n, heads, ratio, ffn = od.ARCHS[fix['kwargs']['backbone_type']]
        return od.init_state(fix['seed'], c, n, heads, ratio, ffn, out_planes=256, prefix='backbone.'), heads, 'backbone.'
    k = fix['kwargs']
    return od.init_state(fix['seed'], k['embedding_planes'], k['block_nums'], k['head_nums'], 4, 'mlp'), k['head_nums'], ''


def test_fixtures_present():
    assert {os.path.basename(p)[:-4] for p in CASES} == set(make_golden.CASES)


@pytest.mark.parametrize('path', CASES, ids=[os.path.basename(p) for p in CASES])
def test_oracle_reproduces_reference_fixture(path):
    from oracle import dinov3 as od
    fix = torch.load(path, weights_only=False)
    torch.set_num_threads(1)
    sd, heads, prefix = oracle_state(fix)
    assert list(sd) == fix['keys']
    torch.manual_seed(fix['draw_seed'])
    assert torch.equal(od.draw_rescale(2), fix['rescale'])
    assert torch.equal(torch.get_rng_state(), fix['rng_after'])
    out, loss, grads = od.loss_and_grads(sd, fix['x'], fix['target'], heads, rescale=fix['rescale'], prefix=prefix)
    torch.testing.assert_close(out, fix['out'], rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(loss, fix['loss'], rtol=1e-5, atol=1e-7)
    assert set(grads) == set(fix['grad_norm'])
    for n, g in grads.items():
        assert abs(g.norm().item() - fix['grad_norm'][n]) <= 1e-4 * max(1e-3, fix['grad_norm'][n]), n
        torch.testing.assert_close(g.flatten()[make_golden.sample_index(g.numel())], fix['grad_sample'][n], rtol=1e-4,
                                   atol=1e-4 * max(1e-6, fix['grad_norm'][n]), msg=n)
    with torch.no_grad():
        ev = od.forward(sd, fix['x'], heads, rescale=None, prefix=prefix)
    torch.testing.assert_close(ev, fix['eval_out'], rtol=1e-5, atol=2e-5)


def _init_digest(sd):
    return {k: (tuple(v.shape), v.double().sum().item(), v.double().square().sum().item()) for k, v in sd.items()}


@pytest.mark.parametrize('arch', BUILT)
def test_backbone_shell_layout_and_init_match_oracle(arch):
    from oracle import dinov3 as od
    from simpleaicv_pytorch_training_examples_b200.detection.models import backbones
    torch.manual_seed(7)
    m = backbones.__dict__[arch]()
    assert m.out_channels == od.ARCHS[arch][0]
    sd = m.state_dict()
    osd = od.init_state(7, *od.ARCHS[arch])
    assert list(sd) == list(osd)
    assert all(torch.equal(sd[k], osd[k]) for k in sd)
    for i in range(len(m.blocks)):
        assert f'blocks.{i}.attn.qkv.bias_mask' in sd and f'blocks.{i}.ls1.gamma' in sd and f'blocks.{i}.ls2.gamma' in sd


@needs_ref
@pytest.mark.parametrize('arch', BUILT)
def test_backbone_shell_layout_and_init_match_live_reference(arch):
    from simpleaicv_pytorch_training_examples_b200.detection.models import backbones
    ref_bb = ref_import.module('SimpleAICV.detection.models.backbones')
    torch.manual_seed(7)
    rs = ref_bb.__dict__[arch]().state_dict()
    torch.manual_seed(7)
    sd = backbones.__dict__[arch]().state_dict()
    assert list(rs) == list(sd)
    assert _init_digest(rs) == _init_digest(sd)


@needs_ref
def test_encoder_and_distill_model_layout_match_live_reference():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    ref_dm = ref_import.module('SimpleAICV.interactive_segmentation.distill_model')
    tea = dict(distill_model.SAM_H_TEACHER, image_size=64, block_nums=2, global_attn_indexes=[1])
    stu = dict(distill_model.DINOV3_B_STUDENT, image_size=64, backbone_type='dinov3_vit_small_patch16_backbone')
    torch.manual_seed(2)
    rs = ref_dm.DINOV3ImageEncoderDistillModel(teacher_params=tea, student_params=stu).state_dict()
    torch.manual_seed(2)
    m = distill_model.DINOV3ImageEncoderDistillModel(teacher_params=tea, student_params=stu)
    sd = m.state_dict()
    assert list(rs) == list(sd) and all(torch.equal(rs[k], sd[k]) for k in rs)
    assert all(not p.requires_grad for p in m.teacher.parameters()) and all(p.requires_grad for p in m.student.parameters())
    assert m.grad_sink() is m.student.grad_sink()


def test_rescale_draw_consumes_cpu_generator_like_reference():
    """The runtime's RoPE table draws its rescale factor exactly as the reference: one CPU draw per training table, none in
    eval; the resulting generator state and coordinates are the reference's."""
    from oracle import dinov3 as od
    from simpleaicv_pytorch_training_examples_b200.engine.dinov3 import rope_sincos
    from simpleaicv_pytorch_training_examples_b200.detection.models import backbones
    m = backbones.dinov3_vit_small_patch16_backbone()
    torch.manual_seed(21)
    want_fac = od.draw_rescale(2)
    want_state = torch.get_rng_state()
    torch.manual_seed(21)
    sin, cos = rope_sincos(m.rope_embed, 5, 3, True)
    assert torch.equal(torch.get_rng_state(), want_state)
    ws, wc = od.rope_table(m.rope_embed.periods, 5, 3, want_fac)
    assert torch.equal(sin, ws) and torch.equal(cos, wc)
    before = torch.get_rng_state()
    sin, cos = rope_sincos(m.rope_embed, 5, 3, False)
    assert torch.equal(torch.get_rng_state(), before)
    ws, wc = od.rope_table(m.rope_embed.periods, 5, 3, None)
    assert torch.equal(sin, ws) and torch.equal(cos, wc)


@needs_ref
def test_rescale_draw_matches_live_reference_module():
    from simpleaicv_pytorch_training_examples_b200.detection.models import backbones
    ref_bb = ref_import.module('SimpleAICV.detection.models.backbones')
    ref = ref_bb.dinov3_vit_small_patch16_backbone().rope_embed.train()
    mine = backbones.dinov3_vit_small_patch16_backbone().rope_embed.train()
    torch.manual_seed(5)
    rs, rc = ref(H=4, W=6)
    state = torch.get_rng_state()
    torch.manual_seed(5)
    ms, mc = mine(4, 6)
    assert torch.equal(torch.get_rng_state(), state) and torch.equal(rs, ms) and torch.equal(rc, mc)


def test_refusals():
    from simpleaicv_pytorch_training_examples_b200.detection.models import backbones
    from simpleaicv_pytorch_training_examples_b200.detection.models.backbones import dinov3vit
    with pytest.raises(NotImplementedError, match='drop_path_rate'):
        backbones.dinov3_vit_small_patch16_backbone(drop_path_rate=0.1)
    with pytest.raises(NotImplementedError, match='shift_coords'):
        backbones.dinov3_vit_small_patch16_backbone(pos_embed_rope_shift_coords=0.1)
    with pytest.raises(NotImplementedError, match='jitter_coords'):
        backbones.dinov3_vit_small_patch16_backbone(pos_embed_rope_jitter_coords=1.5)
    with pytest.raises(NotImplementedError, match='4096'):
        backbones.dinov3_vit_7b_patch16_backbone()
    assert 'dinov3_vit_7b_patch16_backbone' in backbones.__dict__
    with pytest.raises(NotImplementedError):
        dinov3vit.DinoVisionTransformer(embedding_planes=384, block_nums=1, head_nums=6, ffn_layer='swiglu64')
    with pytest.raises(RuntimeError, match='GPU'):
        backbones.dinov3_vit_small_patch16_backbone()(torch.zeros(1, 3, 32, 32))


def test_distill_loss_matches_reference_formula():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.distill_losses import MSELoss
    g = torch.Generator().manual_seed(0)
    t, s = torch.randn(2, 8, 4, 4, generator=g), torch.randn(2, 8, 4, 4, generator=g)
    out = MSELoss()(t, s)
    assert list(out) == ['distill_mse_loss'] and torch.equal(out['distill_mse_loss'], ((s - t) ** 2).mean())


@pytest.mark.parametrize('arch', ['dinov3_vit_small_patch16_backbone', 'dinov3_vit_small_plus_patch16_backbone'])
def test_runtime_lists_every_gemm_weight_once_in_launch_order(arch):
    import test_operands_cpu
    from simpleaicv_pytorch_training_examples_b200.engine.operands import CONV, ROWS, STEM
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.dinov3_segment_anything import DINOV3ViTImageEncoder
    torch.manual_seed(0)
    model = DINOV3ViTImageEncoder(arch, image_size=64)
    ops = model._runtime().operands()
    names = {id(p): n for n, p in model.named_parameters()}
    listed = [names.get(id(op.param)) for op in ops]
    assert None not in listed and len(set(listed)) == len(listed)
    assert set(listed) == test_operands_cpu._gemm_weights(model)
    assert all(op.w is None for op in ops), 'building the runtime allocated an operand copy'
    ffn = ['w1', 'w2', 'w3'] if 'plus' in arch else ['fc1', 'fc2']
    want = []
    for i in range(len(model.backbone.blocks)):
        want += [(f'backbone.blocks.{i}.attn.qkv.weight', ROWS), (f'backbone.blocks.{i}.attn.proj.weight', ROWS)]
        want += [(f'backbone.blocks.{i}.mlp.{n}.weight', ROWS) for n in ffn]
    want += [('backbone.patch_embed.proj.weight', STEM), ('neck.0.weight', ROWS), ('neck.2.weight', CONV)]
    assert [(names[id(op.param)], op.layout) for op in ops] == want
