"""Model constructors with the reference's names (``backbones.__dict__[name](**kwargs)``,
SimpleAICV/classification/backbones/__init__.py) executing on libsaicv_b200.so."""
from .convformer import *  # noqa: F401,F403
from .darknet import *  # noqa: F401,F403
from .resnet import *  # noqa: F401,F403
from .resnetforcifar import *  # noqa: F401,F403
from .van import *  # noqa: F401,F403
from .vit import *  # noqa: F401,F403
