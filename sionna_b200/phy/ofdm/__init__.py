"""OFDM (mirror of sionna.phy.ofdm for the hot path)."""
from .pilot_pattern import PilotPattern, EmptyPilotPattern, KroneckerPilotPattern
from .resource_grid import ResourceGrid, ResourceGridMapper, ResourceGridDemapper, RemoveNulledSubcarriers
from .modulator import OFDMModulator
from .demodulator import OFDMDemodulator
from .channel_estimation import (BaseChannelEstimator, BaseChannelInterpolator, LSChannelEstimator,
                                 NearestNeighborInterpolator, LinearInterpolator)
from .equalization import OFDMEqualizer, LMMSEEqualizer, ZFEqualizer, MFEqualizer
from .precoding import RZFPrecoder, PrecodedChannel, RZFPrecodedChannel, CBFPrecodedChannel, EyePrecodedChannel
from .detection import (LinearDetector, MaximumLikelihoodDetector, MaximumLikelihoodDetectorWithPrior, KBestDetector,
                        EPDetector, MMSEPICDetector)
from .frontend import FusedLSLinearDetector, fusable, frontend_tables
