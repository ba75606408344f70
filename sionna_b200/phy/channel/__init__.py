"""Channel models and channel application (mirror of sionna.phy.channel, SURVEY.md section 8 rows a / f3)."""
from .awgn import AWGN
from .apply_ofdm_channel import ApplyOFDMChannel
from .tdl import TDL, cir_to_ofdm_channel, subcarrier_frequencies
from .cdl import CDL
from .antenna import AntennaElement, PanelArray, Antenna, AntennaArray
from .time_channel import (time_lag_discrete_time_channel, cir_to_time_channel, time_to_ofdm_channel, ApplyTimeChannel, GenerateOFDMChannel,
                           OFDMChannel, GenerateTimeChannel, TimeChannel)
from .rayleigh_block_fading import RayleighBlockFading
from .spatial_correlation import SpatialCorrelation, KroneckerModel, PerColumnModel
from .flat_fading_channel import GenerateFlatFadingChannel, ApplyFlatFadingChannel, FlatFadingChannel
from .utils import exp_corr_mat, one_ring_corr_mat
