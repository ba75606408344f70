"""Signal module (mirror of /root/reference/src/sionna/phy/signal/__init__.py): filters, windows, up/down-sampling,
convolution, normalised DFTs and the empirical PSD / ACLR, on the kernels of ``csrc/signal.cu`` and the OFDM FFT."""
from .utils import convolve, empirical_psd, empirical_aclr, fft, ifft
from .window import Window, HannWindow, HammingWindow, CustomWindow, BlackmanWindow
from .filter import Filter, RaisedCosineFilter, RootRaisedCosineFilter, CustomFilter, SincFilter
from .upsampling import Upsampling
from .downsampling import Downsampling
