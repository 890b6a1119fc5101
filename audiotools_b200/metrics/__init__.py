"""Functions for comparing AudioSignal objects to one another (ref:audiotools/metrics): the spectral losses
(``spectral``), the waveform distances (``distance``), the quality metrics (``quality``: STOI on the GPU; PESQ and
ViSQOL, which call an external library / binary in the reference, are not ported) and the integrated loudness as a
training loss (``loudness``)."""
from . import distance
from . import loudness
from . import quality
from . import spectral
from .distance import L1Loss
from .distance import SISDRLoss
from .loudness import LoudnessLoss
from .quality import STOILoss
from .spectral import MelSpectrogramLoss
from .spectral import MultiScaleSTFTLoss
from .spectral import PhaseLoss
