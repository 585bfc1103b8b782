from .detr_resnet import *  # noqa: F401,F403
from .dinov3vit import *  # noqa: F401,F403
