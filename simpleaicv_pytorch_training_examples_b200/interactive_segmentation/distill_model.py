"""SAM image-encoder distillation wrappers with the reference's constructor surface
(SimpleAICV/interactive_segmentation/distill_model.py:21-127): a SAM ViT teacher and a SAM ViT or DINOv3 student, both
encoders of THIS package, so both forwards and the student's backward run on the H100 runtime.  A frozen teacher runs
under no_grad and gets no gradients.  ``forward(x)`` returns ``(tea_out, stu_out)``; state_dict keys are ``teacher.*`` and
``student.*``."""
import torch
import torch.nn as nn

from ..classification.common import load_state_dict
from .models.dinov3_segment_anything.dinov3_image_encoder import DINOV3ViTImageEncoder
from .models.segment_anything.image_encoder import ViTImageEncoder

__all__ = [
    'ImageEncoderDistillModel',
    'DINOV3ImageEncoderDistillModel',
]

SAM_H_TEACHER = {'image_size': 1024, 'patch_size': 16, 'inplanes': 3, 'embedding_planes': 1280, 'block_nums': 32, 'head_nums': 16,
                 'mlp_ratio': 4, 'out_planes': 256, 'window_size': 14, 'global_attn_indexes': [7, 15, 23, 31],
                 'use_gradient_checkpoint': False}
SAM_B_STUDENT = {'image_size': 1024, 'patch_size': 16, 'inplanes': 3, 'embedding_planes': 768, 'block_nums': 12, 'head_nums': 12,
                 'mlp_ratio': 4, 'out_planes': 256, 'window_size': 14, 'global_attn_indexes': [2, 5, 8, 11],
                 'use_gradient_checkpoint': False}
DINOV3_B_STUDENT = {'backbone_type': 'dinov3_vit_base_patch16_backbone', 'image_size': 1024, 'out_planes': 256,
                    'use_gradient_checkpoint': False}


class _EncoderDistill(nn.Module):

    def __init__(self, teacher, student, teacher_pretrained_path, student_pretrained_path, freeze_teacher):
        super().__init__()
        self.freeze_teacher = freeze_teacher
        self.teacher = teacher
        self.student = student
        load_state_dict(teacher_pretrained_path, self.teacher)
        load_state_dict(student_pretrained_path, self.student)
        if self.freeze_teacher:
            for m in self.teacher.parameters():
                m.requires_grad = False

    def grad_sink(self):
        """Data parallelism reduces the student's gradients (the frozen teacher has none)."""
        return self.student.grad_sink()

    def forward(self, x):
        if self.freeze_teacher:
            with torch.no_grad():
                tea_out = self.teacher(x)
        else:
            tea_out = self.teacher(x)
        stu_out = self.student(x)
        return tea_out, stu_out


class ImageEncoderDistillModel(_EncoderDistill):

    def __init__(self, teacher_params=SAM_H_TEACHER, student_params=SAM_B_STUDENT, teacher_pretrained_path='', student_pretrained_path='',
                 freeze_teacher=True):
        super().__init__(ViTImageEncoder(**teacher_params), ViTImageEncoder(**student_params), teacher_pretrained_path,
                         student_pretrained_path, freeze_teacher)


class DINOV3ImageEncoderDistillModel(_EncoderDistill):

    def __init__(self, teacher_params=SAM_H_TEACHER, student_params=DINOV3_B_STUDENT, teacher_pretrained_path='',
                 student_pretrained_path='', freeze_teacher=True):
        super().__init__(ViTImageEncoder(**teacher_params), DINOV3ViTImageEncoder(**student_params), teacher_pretrained_path,
                         student_pretrained_path, freeze_teacher)
