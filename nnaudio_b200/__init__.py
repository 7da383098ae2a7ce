"""nnaudio_b200 — H100-native (sm_90a) audio -> spectrogram engine with the
``nnAudio.features`` module API.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"

from . import design  # noqa: F401  (host-side basis design; no CUDA needed)
from . import features  # noqa: F401
from .features import *  # noqa: F401,F403
