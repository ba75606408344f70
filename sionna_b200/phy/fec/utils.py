"""FEC test utilities (mirror of parts of /root/reference/src/sionna/phy/fec/utils.py needed by the LDPC tests)."""
import os
import numpy as np
import torch

from ..block import Block
from ..config import config
from .._lib_helpers import philox_fill


class GaussianPriorSource(Block):
    """Fake LLRs of an all-zero codeword sent with BPSK over AWGN (fec/utils.py:16-114): logits ~ N(-mu, sigma^2),
    sigma^2 = 4/no, mu = sigma^2/2. ``call(output_shape, no)``."""

    def __init__(self, *, precision=None, **kwargs):
        super().__init__(precision=precision, **kwargs)

    def __call__(self, output_shape, no=None, mi=None):
        return self._invoke(output_shape, no, mi)

    def call(self, output_shape, no=None, mi=None):
        if no is None:
            if mi is None:
                raise ValueError("Either no or mi must be provided.")
            # mutual-information parametrisation (fec/utils.py:88-96): mu = J^-1(mi), sigma^2 = 2 mu
            mi = float(torch.as_tensor(mi).reshape(-1)[0]) if not isinstance(mi, (int, float)) else float(mi)
            mi = min(max(mi, 1e-7), 1.0)
            mu_llr = float(j_fun_inv(mi))
            sigma_llr = np.sqrt(2 * mu_llr)
        else:
            no = float(torch.as_tensor(no).reshape(-1)[0]) if not isinstance(no, (int, float)) else float(no)
            no = max(no, 1e-7)
            sigma_llr = np.sqrt(4.0 / no)
            mu_llr = sigma_llr ** 2 / 2
        shape = [int(s) for s in output_shape]
        return philox_fill("sb_normal", shape, -mu_llr, sigma_llr, self.device).to(self.rdtype)


def llr2mi(llr, s=None, reduce_dims=True):
    r"""Mutual information estimate :math:`1 - E[\log_2(1 + e^{llr})]` for logits of an all-zero codeword (or of the
    codeword with BPSK signs ``s``), fec/utils.py:116-182. An analysis helper (EXIT charts), not on the hot path."""
    llr = torch.as_tensor(llr)
    if not llr.dtype.is_floating_point:
        raise TypeError("Dtype of llr must be a real-valued float.")
    z = llr if s is None else torch.as_tensor(s).to(llr.dtype) * llr
    z = torch.clamp(z, -100.0, 100.0)
    x = torch.log2(1.0 + torch.exp(z))
    return 1.0 - (x.mean() if reduce_dims else x.mean(dim=-1))


_H1, _H2, _H3 = 0.3073, 0.8935, 1.1064


def j_fun(mu):
    r"""J-function (Brannstrom approximation), fec/utils.py:184-225: mutual information of Gaussian LLRs with mean mu."""
    mu = np.minimum(np.maximum(np.asarray(mu, dtype=np.float64), 1e-10), 1000.0)
    return (1 - 2 ** (-_H1 * (2 * mu) ** _H2)) ** _H3


def j_fun_inv(mi):
    r"""Inverse J-function, fec/utils.py:227-267 (output clipped to 20)."""
    mi = np.minimum(np.maximum(np.asarray(mi, dtype=np.float64), 1e-10), 1.0)
    with np.errstate(divide="ignore"):
        mu = 0.5 * ((-1 / _H1) * np.log2(1 - mi ** (1 / _H3))) ** (1 / _H2)
    return np.minimum(mu, 20.0)


def load_parity_check_examples(pcm_id, verbose=False):
    """Built-in example parity-check matrices (fec/utils.py:478-531): 0 = (7,4) Hamming, 1 = BCH(63,45),
    2 = BCH(127,106), 3 = (3,6)-regular LDPC n=100, 4 = 802.11n LDPC n=648. Returns ``pcm, k, n, coderate``."""
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldpc", "codes", "example_pcms.npz")
    with np.load(p) as d:
        pcm = np.array(d[f"pcm{int(pcm_id)}"], dtype=np.int64)
    n = int(pcm.shape[1])
    k = int(n - pcm.shape[0])
    coderate = k / n
    if verbose:
        print(f"\nn: {n}, k: {k}, coderate: {coderate:.3f}")
    return pcm, k, n, coderate


def bin2int(arr):
    """Integer of a binary sequence, most significant bit first (fec/utils.py:532-549): ``[1, 0, 1]`` -> 5; None for
    an empty sequence."""
    if len(arr) == 0:
        return None
    return int("".join(str(int(x)) for x in arr), 2)


def int2bin(num, length):
    """The ``length`` least significant bits of ``num``, most significant first (fec/utils.py:576-611):
    ``int2bin(5, 4)`` -> ``[0, 1, 0, 1]``, ``int2bin(12, 3)`` -> ``[1, 0, 0]``."""
    assert num >= 0, "Input integer should be non-negative"
    assert length >= 0, "length should be non-negative"
    bits = format(num, f"0{length}b")
    return [int(x) for x in bits[-length:]] if length else []
