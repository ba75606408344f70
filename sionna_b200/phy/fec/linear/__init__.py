"""Binary linear block codes (mirror of sionna.phy.fec.linear): generic generator-matrix encoding and ordered
statistics decoding."""
from .encoding import LinearEncoder
from .decoding import OSDecoder
