"""Small wrappers around C-ABI calls shared by several blocks."""
import torch

from .config import config
from .._lib import lib, check, ptr, current_stream


def philox_fill(fn, shape, a, b, device):
    """float32 tensor of ``shape`` drawn by ``fn`` (``"sb_normal"``: a + b * N(0,1); ``"sb_uniform"``: uniform in [a, b))
    from the global Philox stream."""
    out = torch.empty([int(v) for v in shape], dtype=torch.float32, device=device)
    seed, off = config.next_philox()
    check(getattr(lib(), fn)(ptr(out), out.numel(), float(a), float(b), seed, off, current_stream()), fn)
    return out
