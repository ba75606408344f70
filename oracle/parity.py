"""The parity toolkit of the kernel tests (DESIGN §4): the single-precision error envelope, the one definition of the
bar for kernels that are not bit-exact, and the inputs the tests share. The bars themselves stay in the test files.
Every generator draws from the caller's `rng` in a fixed order, so a test's seed fixes its inputs."""
import numpy as np


# ---- the envelope -----------------------------------------------------------------------------------------------------
def rel_err(got, ref, axis=-1, scale=None):
    """|got - ref| relative to the rms of ref along `axis` (an int, a tuple, or None for the whole array), or to a
    given `scale` (broadcast against ref; np.abs(ref) for errors relative per element). Entries where ref is not
    finite count as zero error and as zero in the rms."""
    fin = np.isfinite(ref)
    if scale is None:
        scale = np.sqrt(np.mean(np.abs(np.where(fin, ref, 0)) ** 2, axis=axis, keepdims=True))
    with np.errstate(invalid="ignore"):                   # inf - inf at masked entries
        return np.where(fin, np.abs(got - ref), 0) / np.maximum(scale, 1e-30)


def envelope(what, got, f32, ref, bar, floor=(0.0, 0.0), **rel_err_kw):
    """'' if got's (the kernel's) error is within bar = (rms, max) times f32's (the complex64 evaluation's), both
    against ref, else the measurement line, which is printed either way. got and f32 must be finite exactly where ref
    is. floor = (rms, max): the least complex64 error the bar applies to. rel_err_kw go to `rel_err`."""
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin), f"{what}: kernel finite where the oracle is not (or vice versa)"
    assert np.array_equal(np.isfinite(f32), fin), f"{what}: complex64 evaluation finite where the oracle is not (or vice versa)"
    a, b = rel_err(got, ref, **rel_err_kw), rel_err(f32, ref, **rel_err_kw)
    rms_a, max_a = float(np.sqrt(np.mean(a ** 2))), float(a.max())
    rms_b, max_b = max(float(np.sqrt(np.mean(b ** 2))), floor[0]), max(float(b.max()), floor[1])
    line = (f"{what}: kernel rms {rms_a:.2e} max {max_a:.2e} | complex64 rms {rms_b:.2e} max {max_b:.2e} "
            f"| ratio rms {rms_a / max(rms_b, 1e-30):.2f} max {max_a / max(max_b, 1e-30):.2f} "
            f"(bar {bar[0]:g} / {bar[1]:g})")
    print(line)
    return "" if rms_a <= bar[0] * rms_b and max_a <= bar[1] * max_b else line


# ---- MIMO inputs ------------------------------------------------------------------------------------------------------
def cnormal(rng, shape, scale=1.0, dtype=np.complex64):
    """CN(0, scale^2) samples: real parts drawn first, then imaginary parts."""
    return ((rng.normal(size=shape) + 1j * rng.normal(size=shape)) * scale / np.sqrt(2)).astype(dtype)


def noise_covariance(rng, num, m, no):
    """num well-conditioned, non-diagonal noise covariances no * (I + 0.5 A A^H / m), complex64."""
    a = cnormal(rng, (num, m, m))
    return (no * (np.eye(m) + 0.5 * a @ np.conj(np.swapaxes(a, -1, -2)) / m)).astype(np.complex64)


def mimo_problem(rng, num, m, k, points, no, return_indices=False):
    """num problems y = H x + n, x drawn uniformly from `points`, n ~ CN(0, S) with S = noise_covariance(no):
    (y, h, s) with y [num, m], h [num, m, k], s [num, m, m] complex64, and the indices of x [num, k] if asked."""
    h = cnormal(rng, (num, m, k))
    ind = rng.integers(0, len(points), (num, k))
    s = noise_covariance(rng, num, m, no)
    n = (np.linalg.cholesky(s.astype(np.complex128)) @ cnormal(rng, (num, m, 1)))[..., 0]
    y = ((h @ points[ind][..., None])[..., 0] + n).astype(np.complex64)
    return (y, h, s, ind) if return_indices else (y, h, s)


def constellation(kind, m):
    """A Constellation of 2^m points: "qam" / "pam", or "custom" (fixed random points, normalised and centred)."""
    from sionna_b200.phy.mapping import Constellation
    if kind == "custom":
        rng = np.random.default_rng(99)
        pts = (rng.normal(size=2 ** m) + 1j * rng.normal(size=2 ** m)).astype(np.complex64)
        return Constellation("custom", m, points=pts, normalize=True, center=True)
    return Constellation(kind, m)


def ofdm_detection_case(cfg, rng, no_range, ev_shape=None, no_shape=None):
    """(rg, sm, oracle stream dict, y_eff, h, err_var, no, points) of an OFDM detection problem on a 3-symbol Kronecker
    grid (symbol 1 pilots), cfg = (name, batch, num_tx, streams per tx, num_rx, rx antennas, bits per symbol,
    association, ...). The noise variance is drawn uniformly from no_range per (batch, rx, antenna); no_shape () takes
    0.1 instead, another shape the leading entries of the draw. err_var has ev_shape (default: h's), () for 0.005."""
    from oracle import mapping as MAP
    from oracle import ofdm as F
    from sionna_b200.phy.ofdm import ResourceGrid
    from sionna_b200.phy.mimo import StreamManagement
    name, b, num_tx, spt, rx, ant, m, assoc = cfg[:8]
    s_ = 3
    txs = num_tx * spt
    f_ = txs * max(1, round(12 / txs))
    rg = ResourceGrid(s_, f_, 15e3, num_tx=num_tx, num_streams_per_tx=spt, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[1])
    sm = StreamManagement(np.array(assoc), spt)
    pts = MAP.qam(m).astype(np.complex64)
    h = cnormal(rng, (b, rx, ant, num_tx, spt, s_, f_))
    x = pts[rng.integers(0, len(pts), (b, num_tx, spt, s_, f_))]
    no = rng.uniform(*no_range, size=(b, rx, ant)).astype(np.float32)
    if no_shape == ():
        no = np.float32(0.1)
    elif no_shape is not None:
        no = no[(slice(None),) * len(no_shape) + (0,) * (3 - len(no_shape))].reshape(no_shape)
    no_b = np.broadcast_to(np.asarray(no).reshape(np.shape(no) + (1,) * (3 - np.ndim(no))), (b, rx, ant))
    y = np.einsum("brmtksf,btksf->brmsf", h.astype(np.complex128), x)
    y = (y + cnormal(rng, y.shape) * np.sqrt(no_b)[..., None, None]).astype(np.complex64)
    ev_shape = h.shape if ev_shape is None else ev_shape
    ev = (0.01 * rng.uniform(size=ev_shape)).astype(np.float32) if ev_shape else np.float32(0.005)
    return rg, sm, F.stream_management(assoc, spt), y, h, ev, no, pts


# ---- LDPC inputs and checks -------------------------------------------------------------------------------------------
def bpsk_llr(c, ebno_db, rate, rng):
    """Channel LLRs (float32) of codewords c [B, n] sent as BPSK (bit 1 -> +1) over AWGN at Eb/N0 ebno_db [B] (dB) and
    code rate `rate`. c = np.zeros((B, n)) gives the all-zero codeword."""
    no = 1.0 / (10 ** (np.asarray(ebno_db)[:, None] / 10) * rate)
    y = (2.0 * c - 1.0) + rng.normal(size=c.shape) * np.sqrt(no / 2)
    return (4 * y / no).astype(np.float32)


def lifted_pcm(z, rows, cols, last, br, bc, sh):
    """Parity-check matrix (float64) of the base graph with entries (br, bc) and shifts sh lifted by z: entry (r, c, s)
    connects check r z + i to variable c z + (i + s) mod z. The last block row is cut to `last` checks."""
    pcm = np.zeros((rows * z, cols * z), np.float64)
    i = np.arange(z)
    for r, c, s in zip(br, bc, sh):
        pcm[r * z + i, c * z + (i + s) % z] = 1
    return pcm[:(rows - 1) * z + last]


def assert_bit_exact(x, st, xr, sr):
    """Soft outputs x and state st (device tensors) equal the oracle's xr, sr bit for bit."""
    assert np.array_equal(x.cpu().numpy(), xr)
    assert np.array_equal(st.cpu().numpy(), sr)


def assert_mixed_convergence(xr, c, groups):
    """The batch, `groups` equal Eb/N0 groups in ascending order, holds codewords that fail (in the first group) and
    only converged ones (in the last): soft outputs xr against the codewords c."""
    err = ((xr > 0) != (c > 0)).any(axis=1)
    g = len(err) // groups
    assert err[:g].any() and not err[-g:].any()
