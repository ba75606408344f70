"""Forward error correction (mirror of sionna.phy.fec): LDPC, convolutional and turbo codes, interleavers, CRC,
scrambling and test utilities."""
from . import ldpc
from . import conv
from . import interleaving
from . import turbo
from . import utils
from . import crc
from . import scrambling
from .crc import CRCEncoder, CRCDecoder
from .scrambling import TB5GScrambler, Scrambler, Descrambler
