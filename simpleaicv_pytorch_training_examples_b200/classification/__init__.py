"""Drop-in counterpart of ``SimpleAICV.classification`` for the H100 hot path: ``backbones``
(model constructors with the reference's names and state_dict layout) and ``losses``."""
from . import backbones, losses  # noqa: F401
