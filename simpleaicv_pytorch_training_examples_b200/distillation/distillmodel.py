"""Knowledge-distillation wrapper (SURVEY.md 8 f4) with the reference's constructor surface
(SimpleAICV/distillation/distillmodel.py:19-60): teacher and student are backbones of THIS package (so both forwards,
and the student's backward, run on the H100 runtime), the teacher is frozen and evaluated without a tape.
``forward(x)`` returns ``(tea_out, stu_out)``."""
import torch
import torch.nn as nn

from ..classification import backbones
from ..classification.common import load_state_dict

__all__ = ['KDModel']


class KDModel(nn.Module):

    def __init__(self, teacher_type='resnet34', student_type='resnet18', teacher_pretrained_path='', student_pretrained_path='',
                 freeze_teacher=True, num_classes=1000, use_gradient_checkpoint=False):
        super().__init__()
        self.freeze_teacher = freeze_teacher
        self.teacher = backbones.__dict__[teacher_type](**{'num_classes': num_classes, 'use_gradient_checkpoint': use_gradient_checkpoint})
        self.student = backbones.__dict__[student_type](**{'num_classes': num_classes, 'use_gradient_checkpoint': use_gradient_checkpoint})
        load_state_dict(teacher_pretrained_path, self.teacher)
        load_state_dict(student_pretrained_path, self.student)
        if self.freeze_teacher:
            for m in self.teacher.parameters():
                m.requires_grad = False

    def grad_sink(self):
        """Where data parallelism collects the gradients: the student's sink, and the teacher's as well when it is trained
        (its runtime writes its gradients through a sink of its own)."""
        if self.freeze_teacher:
            return self.student.grad_sink()
        return [self.teacher.grad_sink(), self.student.grad_sink()]

    def forward(self, x):
        if self.freeze_teacher:
            with torch.no_grad():
                tea_out = self.teacher(x)
        else:
            tea_out = self.teacher(x)
        stu_out = self.student(x)
        return tea_out, stu_out
