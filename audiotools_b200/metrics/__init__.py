"""Functions for comparing AudioSignal objects to one another (ref:audiotools/metrics): the spectral losses
(``spectral``) and the waveform distances (``distance``).  ``quality`` (STOI / PESQ / ViSQOL) is not ported."""
from . import distance
from . import spectral
from .distance import L1Loss
from .distance import SISDRLoss
from .spectral import MelSpectrogramLoss
from .spectral import MultiScaleSTFTLoss
from .spectral import PhaseLoss
