"""Interleavers on the GPU (sb_gather_rows): the reference's TestRandomInterleaver, TestDeinterleaver and
TestTurbo3GPPInterleaver cases that do not depend on TensorFlow's random draws, restated."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _il():
    from sionna_b200.phy.fec import interleaving
    return interleaving


def test_random_sequence_and_inverse(cuda_device):
    il = _il()
    x = torch.arange(1000, dtype=torch.float32, device="cuda").repeat(4, 1)
    for keep_batch in (True, False):
        inter = il.RandomInterleaver(seed=7, keep_batch_constant=keep_batch)
        y = inter(x)
        assert tuple(y.shape) == (4, 1000)
        assert all(torch.equal(torch.sort(r)[0], x[0]) for r in y)        # a permutation of each row
        assert not torch.equal(y, x)
        assert torch.equal(inter(y, inverse=True), x)
        assert torch.equal(il.Deinterleaver(inter)(y), x)
        assert torch.equal(y[0], y[1]) == keep_batch                     # one permutation, or one per example
        assert torch.equal(inter(x), y)                                   # keep_state: the same permutation again


def test_random_seed(cuda_device):
    il = _il()
    x = torch.arange(100, dtype=torch.float32, device="cuda").repeat(2, 1)
    a, b = il.RandomInterleaver(seed=1), il.RandomInterleaver(seed=1)
    assert torch.equal(a(x), b(x))
    assert not torch.equal(a(x), il.RandomInterleaver(seed=2)(x))
    assert torch.equal(a(x, seed=5), il.RandomInterleaver(seed=5)(x))
    assert torch.equal(il.Deinterleaver(a)(a(x, seed=9), seed=9), x)
    c = il.RandomInterleaver(keep_state=False)
    assert not torch.equal(c(x), c(x))
    with pytest.raises(ValueError):
        c(x, inverse=True)
    from sionna_b200.phy import config
    config.seed = 3
    d = il.RandomInterleaver()
    config.seed = 3
    assert il.RandomInterleaver().seed == d.seed


@pytest.mark.parametrize("axis", (-1, 1, 2, -2))
def test_multi_dim_and_axis(cuda_device, axis):
    il = _il()
    x = torch.randn(3, 5, 7, 11, device="cuda")
    for inter in (il.RandomInterleaver(seed=4, axis=axis), il.Turbo3GPPInterleaver(axis=axis)):
        y = inter(x)
        n = x.shape[axis]
        p = inter.perm(n) if isinstance(inter, il.Turbo3GPPInterleaver) else inter.perm(n)[0]
        ref = torch.index_select(x, axis % 4, torch.from_numpy(p).cuda())
        assert torch.equal(y, ref)
        assert torch.equal(il.Deinterleaver(inter)(y), x)


def test_invalid_shapes_and_args(cuda_device):
    il = _il()
    with pytest.raises(ValueError):
        il.RandomInterleaver(axis=3)(torch.zeros(2, 4, device="cuda"))
    with pytest.raises(ValueError):
        il.Turbo3GPPInterleaver(axis=3)(torch.zeros(2, 4, device="cuda"))
    with pytest.raises(ValueError):
        il.Turbo3GPPInterleaver()(torch.zeros(2, 6145, device="cuda"))
    with pytest.raises(TypeError):
        il.RandomInterleaver(seed=1.5)
    with pytest.raises(TypeError):
        il.RandomInterleaver(keep_batch_constant=1)
    with pytest.raises(TypeError):
        il.Turbo3GPPInterleaver(inverse=1)
    with pytest.raises(ValueError):
        il.Deinterleaver(object())


@pytest.mark.parametrize("dtype", (torch.float32, torch.float64, torch.int32, torch.int64, torch.complex64,
                                   torch.complex128))
def test_dtype(cuda_device, dtype):
    il = _il()
    x = (torch.arange(2 * 50, device="cuda") % 97).reshape(2, 50).to(dtype)
    prec = "double" if dtype in (torch.float64, torch.complex128) else "single"      # floats are cast to the precision
    for inter in (il.RandomInterleaver(seed=3, precision=prec), il.Turbo3GPPInterleaver(precision=prec)):
        y = inter(x)
        assert y.dtype == dtype
        assert torch.equal(il.Deinterleaver(inter)(y), x)
    with pytest.raises(TypeError):
        il.Turbo3GPPInterleaver()(torch.zeros(2, 40, dtype=torch.int16, device="cuda"))


def test_turbo3gpp_sequence(cuda_device):
    """TestTurbo3GPPInterleaver.test_sequence_dimension / test_inverse: the QPP permutation of TS 36.212 for k = 40
    (f1 = 3, f2 = 10), and shortened lengths."""
    il = _il()
    inter = il.Turbo3GPPInterleaver()
    x = torch.arange(40, dtype=torch.float32, device="cuda")[None]
    i = np.arange(40)
    assert np.array_equal(inter(x)[0].cpu().numpy(), (3 * i + 10 * i * i) % 40)
    for k in (41, 500, 6144):
        x = torch.randn(3, k, device="cuda")
        y = inter(x)
        assert torch.equal(inter(y, inverse=True), x)
        assert torch.equal(il.Deinterleaver(inter)(y), x)
