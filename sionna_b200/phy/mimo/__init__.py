"""MIMO (mirror of sionna.phy.mimo for the hot path): stream management, RZF / CBF precoding, LMMSE / ZF / MF equalisation, linear, maximum-likelihood, K-Best, EP and MMSE-PIC detection."""
from .stream_management import StreamManagement
from .precoding import rzf_precoding_matrix, cbf_precoding_matrix, rzf_precoder
from .equalization import lmmse_equalizer, lmmse_matrix, zf_equalizer, mf_equalizer
from .utils import whiten_channel
from .detection import (LinearDetector, MaximumLikelihoodDetector, KBestDetector, List2LLR, List2LLRSimple,
                        EPDetector, MMSEPICDetector)
