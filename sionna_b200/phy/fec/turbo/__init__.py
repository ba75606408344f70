"""Turbo codes (mirror of sionna.phy.fec.turbo): ``TurboEncoder`` composed of the interleaving and convolutional
kernels, ``TurboDecoder`` on the fused kernel of ``csrc/conv.cu``; ``TurboTermination``, ``polynomial_selector`` and
``puncture_pattern`` on the host."""
from .encoding import TurboEncoder
from .decoding import TurboDecoder
from .utils import TurboTermination, polynomial_selector, puncture_pattern
