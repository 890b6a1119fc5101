"""audiotools_b200 -- H100-native (sm_90a) engine for the AudioSignal transform/augment hot
path of descriptinc/audiotools, behind the reference's own method surface::

    from audiotools_b200 import AudioSignal
    from audiotools_b200.data import transforms as tfm

The DSP runs in ``audiotools_b200/csrc/libb2a.so`` (hand-written CUDA, C ABI in
``include/b2a.h``); there is no CPU implementation and no fallback.
"""
__version__ = "0.1.0"
from .core import AudioSignal
from .core import STFTParams
from .core import Meter
from .core import util
from . import data
from . import metrics
from . import ml
from .data import transforms
