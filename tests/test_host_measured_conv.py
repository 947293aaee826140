"""CPU tests (no GPU) of the projection from convolution measurements: ConvOperator's geometry, application and CSR form
against a float64 conv2d, its constructors against the test operators, the sizers' refusals without a handle, and
DefenseGANBase's checks before any native call."""
import ctypes
import os

import numpy as np
import pytest
import torch

import measured_oracle as MO
import sparse_operators as SO



def test_conv_op_m_and_sizer_refuse_bad_geometry_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    for op in (_native.dgan_conv_op(5, 5, 2, 2, 1), _native.dgan_conv_op(0, 5, 0, 2, 1),
               _native.dgan_conv_op(5, 5, 3, 2, 1), _native.dgan_conv_op(5, 5, 2, 2, 17)):
        assert lib.dgan_conv_op_m(None, ctypes.byref(op)) == 0
        assert lib.dgan_workspace_bytes_measured_conv(None, 2, 2, ctypes.byref(op), None, 0, 0) == 0
    assert lib.dgan_conv_op_m(None, None) == 0
    fn = lib.dgan_debug_workspace_layout_measured_conv
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(_native.dgan_conv_op), ctypes.c_char_p, ctypes.c_int]
    buf = ctypes.create_string_buffer(1 << 12)
    assert fn(None, 4, ctypes.byref(_native.dgan_conv_op(5, 5, 2, 2, 1)), buf, len(buf)) == -1


# ---- ConvOperator ----

def _k(kh, kw, seed, zeros=False):
    k = np.random.RandomState(seed).standard_normal((kh, kw)).astype(np.float32)
    if zeros:
        k.reshape(-1)[::3] = 0.0
    return k


GRID = [  # (kh, kw, padding, stride, zero and negative taps)
    (4, 4, 1, 1, False), (2, 6, (0, 2), 1, False), (3, 5, (0, 2), 2, False), (5, 3, (2, 1), 3, False),
    (1, 1, 0, 1, False), (3, 3, 1, 1, True), (7, 2, (3, 0), 4, True), (2, 2, 0, 2, False),
]


@pytest.mark.parametrize("image_dim", [(28, 28, 1), (10, 13, 3)])
@pytest.mark.parametrize("kh,kw,pad,stride,zeros", GRID)
def test_csr_and_call_equal_float64_conv2d(kh, kw, pad, stride, zeros, image_dim):
    from defensegan_b200.operators import ConvOperator
    h, w, c = image_dim
    op = ConvOperator(_k(kh, kw, kh * 10 + kw, zeros), stride=stride, padding=pad)
    x = torch.tensor(np.random.RandomState(1).standard_normal((2, h, w, c)))
    ph, pw = op.padding
    want = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), op.kernel.double().expand(c, 1, kh, kw), stride=stride,
                                      padding=(ph, pw), groups=c).permute(0, 2, 3, 1).reshape(2, -1)
    ho, wo, _ = op.out_shape(image_dim)
    assert want.shape[1] == ho * wo * c == op.num_measurements(image_dim)
    a = op.to_sparse_csr(image_dim)
    assert a.layout == torch.sparse_csr and a.shape == (ho * wo * c, h * w * c) and a.values().dtype == torch.float32
    crow, col = a.crow_indices(), a.col_indices()
    for r in range(a.shape[0]):                          # columns strictly ascending within each row
        assert bool((col[crow[r] + 1:crow[r + 1]] > col[crow[r]:crow[r + 1] - 1]).all())
    assert not bool((a.values() == 0).any())
    got = (a.to_dense().double() @ x.reshape(2, -1).t()).t()
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(op(x).numpy(), want.numpy(), rtol=1e-12, atol=1e-12)


def test_per_image_kernels():
    from defensegan_b200.operators import ConvOperator
    ks = np.stack([_k(3, 3, i) for i in range(3)])
    op = ConvOperator(ks, stride=2, padding=1)
    assert op.per_image and op.kernels(3).shape == (3, 3, 3)
    x = torch.tensor(np.random.RandomState(2).standard_normal((3, 28, 28, 1)))
    y = op(x)
    for i in range(3):
        one = ConvOperator(ks[i], stride=2, padding=1)
        assert torch.equal(y[i], one(x[i:i + 1])[0])
        assert torch.equal(op.to_sparse_csr((28, 28, 1), image=i).to_dense(), one.to_sparse_csr((28, 28, 1)).to_dense())
    with pytest.raises(ValueError, match="3 per-image kernels for 2 images"):
        op.kernels(2)
    shared = ConvOperator(ks[0])
    assert torch.equal(shared.kernels(4), torch.tensor(ks[0]).expand(4, 3, 3))


def test_constructors_reproduce_the_test_operators():
    from defensegan_b200.operators import ConvOperator
    for dim in ((28, 28, 1), (12, 10, 3)):
        g = ConvOperator.gaussian(5, 1.0)
        assert np.array_equal(g.to_sparse_csr(dim).to_dense().numpy(), SO.blur_operator(*dim))
        b = ConvOperator.box(2)
        assert np.array_equal(b.to_sparse_csr(dim).to_dense().numpy(), MO.block_average_operator(*dim, 2))
    assert np.array_equal(ConvOperator.box(4).to_sparse_csr((28, 28, 1)).to_dense().numpy(),
                          MO.block_average_operator(28, 28, 1, 4))


@pytest.mark.parametrize("kwargs,match", [
    (dict(kernel=np.ones((0, 3))), "kh = 0"), (dict(kernel=np.ones((3, 33))), "kw = 33"),
    (dict(kernel=np.ones(3)), "kernel must be"), (dict(kernel=np.ones((3, 3)), stride=0), "stride = 0"),
    (dict(kernel=np.ones((3, 3)), stride=17), "stride = 17"), (dict(kernel=np.ones((3, 3)), padding=2), "ph = 2"),
    (dict(kernel=np.ones((3, 3)), padding=(1, -1)), "pw = -1"), (dict(kernel=np.ones((3, 3)), padding=(1, 2, 3)), "padding"),
    (dict(kernel=np.full((3, 3), np.nan)), "finite"), (dict(kernel=np.ones((3, 3)), stride=1.5), "stride"),
])
def test_bad_geometry_and_values_are_refused_at_construction(kwargs, match):
    from defensegan_b200.operators import ConvOperator
    with pytest.raises(ValueError, match=match):
        ConvOperator(**kwargs)


def test_a_kernel_larger_than_the_image_is_refused():
    from defensegan_b200.operators import ConvOperator
    with pytest.raises(ValueError, match="does not fit"):
        ConvOperator(np.ones((29, 3))).out_shape((28, 28, 1))


# ---- DefenseGANBase ----

class FakeNative:
    def __init__(self):
        self.calls = []

    def reconstruct_measured(self, y, a, *args, **kw):
        self.calls.append((y, a, args, kw))
        return y


def _gan():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    fake = FakeNative()
    gan._as_cuda = lambda t: (t if isinstance(t, torch.Tensor) else torch.as_tensor(t)).to(torch.float32)
    gan._get_native = lambda device: fake
    return gan, fake


def test_defensegan_passes_the_broadcast_kernel_and_m():
    from defensegan_b200.operators import ConvOperator
    gan, fake = _gan()
    gan.rec_rr, gan.rec_iters, gan.rec_lr = 4, 9, 3.0
    op = ConvOperator.gaussian(5, 1.0)
    y = np.random.RandomState(1).standard_normal((3, 784)).astype(np.float32)
    gan.reconstruct_measured(y, op, batch_size=3, z_row_offset=8, prune=[(5, 2)])
    (yt, at, args, kw), = fake.calls
    assert isinstance(at, ConvOperator) and at.kernel.shape == (3, 5, 5)
    assert torch.equal(at.kernel, op.kernel.expand(3, 5, 5)) and at.stride == 1 and at.padding == (2, 2)
    assert at.num_measurements((28, 28, 1)) == yt.shape[1] == 784
    assert args == (4, 9, 3.0) and kw["z_row_offset"] == 8 and kw["prune"] == [(5, 2)] and kw["seed"] == gan.last_seed


BAD = {
    "per-image kernel count": (lambda C: C(np.ones((3, 5, 5)), padding=2), (2, 784), "3 per-image kernels for 2 images"),
    "measurement count": (lambda C: C.gaussian(5, 1.0), (2, 783), "measurements must be \\[B, 784\\]"),
    "measurement rank": (lambda C: C.box(2), (2, 14, 14), "measurements must be \\[B, 196\\]"),
    "kernel too large": (lambda C: C(np.ones((29, 3))), (2, 784), "does not fit"),
    "non-finite measurements": (lambda C: C.box(2), "nan", "^measurements must be finite"),
    "batch_size": (lambda C: C.box(2), (2, 196), "batch_size"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_bad_inputs_are_refused_before_any_native_call(case):
    from defensegan_b200.operators import ConvOperator
    make, y_shape, match = BAD[case]
    gan, fake = _gan()
    counter = gan._call_counter
    y = np.full((2, 196), np.nan, dtype=np.float32) if y_shape == "nan" else np.ones(y_shape, dtype=np.float32)
    with pytest.raises(ValueError, match=match):
        gan.reconstruct_measured(y, make(ConvOperator), batch_size=3 if case == "batch_size" else None)
    assert fake.calls == [] and gan._call_counter == counter


def test_non_finite_kernels_are_refused_before_any_native_call():
    from defensegan_b200.operators import ConvOperator
    gan, fake = _gan()
    op = ConvOperator(np.ones((3, 3, 3), dtype=np.float32), padding=1)
    op.kernel[1, 1, 1] = float("inf")                # changed after construction
    with pytest.raises(ValueError, match="^operator kernels must be finite"):
        gan.reconstruct_measured(np.ones((3, 784), dtype=np.float32), op)
    assert fake.calls == []
