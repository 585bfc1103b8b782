"""DINOv3 SAM image encoder with the reference's constructor surface and state_dict layout
(SimpleAICV/interactive_segmentation/models/dinov3_segment_anything/dinov3_image_encoder.py:36-75): a DINOv3 ViT backbone
(``backbone.*``) followed by the SAM neck (``neck.*``).  The encoder owns the one runtime (engine.dinov3.DINOv3RT) that
runs backbone and neck forward and backward through one autograd node and one gradient sink."""
import torch.nn as nn

from ....detection.models import backbones
from ....engine.dinov3 import DINOv3RT
from ....engine.runtime import RuntimeModule
from ..segment_anything.image_encoder import LayerNorm2d


class DINOV3ViTImageEncoder(RuntimeModule):

    def __init__(self, backbone_type, backbone_pretrained_path='', image_size=1024, out_planes=256, use_gradient_checkpoint=False):
        super().__init__()
        self.image_size = image_size
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.backbone = backbones.__dict__[backbone_type](**{'pretrained_path': backbone_pretrained_path,
                                                             'use_gradient_checkpoint': use_gradient_checkpoint})
        self.neck = nn.Sequential(
            nn.Conv2d(self.backbone.out_channels, out_planes, kernel_size=1, stride=1, padding=0, bias=False), LayerNorm2d(out_planes),
            nn.Conv2d(out_planes, out_planes, kernel_size=3, stride=1, padding=1, bias=False), LayerNorm2d(out_planes))

    def _build_runtime(self):
        return DINOv3RT(self.backbone, self.neck, neck_checkpoint=self.use_gradient_checkpoint)

    def forward(self, x):
        """x: fp32 [B, 3, S, S] -> fp32 [B, out_planes, S/16, S/16]"""
        return self._run(x.float())
