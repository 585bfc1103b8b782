"""Knowledge-distillation pieces (SURVEY.md 8 f4): the loss tails equal the reference's
(SimpleAICV/distillation/losses.py) on the same logits, values and gradients; KDModel has the reference's layout."""
import pytest
import torch


def _ref_losses():
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    ref_import._ensure_path()
    from SimpleAICV.distillation import losses
    return losses


@pytest.mark.parametrize('name,args', [('KDLoss', (4.0,)), ('DMLLoss', (2.0,)), ('L2Loss', ()), ('CELoss', ()), ('OneHotLabelCELoss', ())])
def test_distillation_losses_match_reference(name, args):
    ref = _ref_losses()
    from simpleaicv_pytorch_training_examples_b200.distillation import losses
    g = torch.Generator().manual_seed(0)
    stu = (torch.randn(16, 100, generator=g) * 3).requires_grad_(True)
    stu2 = stu.detach().clone().requires_grad_(True)
    tea = torch.randn(16, 100, generator=g) * 3
    if name == 'CELoss':
        other = torch.randint(0, 100, (16,), generator=g)
    elif name == 'OneHotLabelCELoss':
        other = torch.softmax(torch.randn(16, 100, generator=g), dim=1)
    else:
        other = tea
    a = getattr(ref, name)(*args)(stu, other)
    b = getattr(losses, name)(*args)(stu2, other)
    a.backward()
    b.backward()
    assert torch.equal(a.detach(), b.detach())
    assert torch.equal(stu.grad, stu2.grad)


def test_kdmodel_layout_and_frozen_teacher():
    from simpleaicv_pytorch_training_examples_b200.distillation.distillmodel import KDModel
    m = KDModel(teacher_type='resnet34', student_type='resnet18', num_classes=10)
    assert all(not p.requires_grad for p in m.teacher.parameters()) and all(p.requires_grad for p in m.student.parameters())
    keys = list(m.state_dict().keys())
    assert keys[0].startswith('teacher.') and any(k.startswith('student.') for k in keys)
    with pytest.raises(RuntimeError, match='no CPU'):
        m(torch.randn(1, 3, 32, 32))
