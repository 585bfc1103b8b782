"""Knowledge distillation on the H100 runtime (SURVEY.md 8 f4): KDModel's frozen teacher runs without a tape, the student's
gradients equal those of the same student trained stand-alone with the same combined loss, and the teacher receives none."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_kd_model_student_gradients_match_a_standalone_student():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.distillation import losses
    from simpleaicv_pytorch_training_examples_b200.distillation.distillmodel import KDModel
    torch.manual_seed(0)
    kd = KDModel(teacher_type='resnet34', student_type='resnet18', num_classes=10).cuda().train()
    kd.teacher.eval()
    x = torch.randn(8, 3, 64, 64, device='cuda')
    y = torch.randint(0, 10, (8,), device='cuda')
    ce, kdl = losses.CELoss(), losses.KDLoss(4.0)
    tea, stu = kd(x)
    assert not tea.requires_grad and stu.requires_grad
    (ce(stu, y) + 0.5 * kdl(stu, tea)).backward()
    assert all(p.grad is None for p in kd.teacher.parameters())
    solo = backbones.resnet18(num_classes=10).cuda().train()
    solo.load_state_dict(kd.student.state_dict())
    out = solo(x)
    (ce(out, y) + 0.5 * kdl(out, tea)).backward()
    torch.cuda.synchronize()
    assert torch.equal(out, stu)
    for (n, p), q in zip(kd.student.named_parameters(), solo.parameters()):
        assert torch.equal(p.grad, q.grad), n       # the runtime is bit-deterministic
