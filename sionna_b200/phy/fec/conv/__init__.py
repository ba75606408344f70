"""Convolutional codes (mirror of sionna.phy.fec.conv): ``ConvEncoder``, ``ViterbiDecoder``, ``BCJRDecoder`` on the
trellis kernels of ``csrc/conv.cu``; ``Trellis`` and ``polynomial_selector`` on the host."""
from .encoding import ConvEncoder
from .decoding import ViterbiDecoder, BCJRDecoder
from .utils import Trellis, polynomial_selector
