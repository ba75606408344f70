"""MIMO (mirror of sionna.phy.mimo for the hot path): stream management, LMMSE equalisation, linear, maximum-likelihood, K-Best, EP and MMSE-PIC detection."""
from .stream_management import StreamManagement
from .equalization import lmmse_equalizer, lmmse_matrix
from .utils import whiten_channel
from .detection import (LinearDetector, MaximumLikelihoodDetector, KBestDetector, List2LLR, List2LLRSimple,
                        EPDetector, MMSEPICDetector)
