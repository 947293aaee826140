"""CPU tests (no GPU) of the projection from sparse linear measurements: the binding's and DefenseGANBase's handling of
sparse operators, the checks that refuse a malformed CSR before any native call, and the test operators."""
import ctypes
import os

import numpy as np
import pytest
import torch

import measured_oracle as MO
import sparse_operators as SO
from oracle import defensegan_oracle as O

from recording import Out, cpu_native  # noqa: F401  (the fixture)


def test_workspace_bytes_measured_csr_refuses_bad_m_and_nnz_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    for m, nnz in ((0, 0), (-1, 0), (785, 10), (10, -1), (1, 785), (2, 2 * 784 + 1)):
        assert lib.dgan_workspace_bytes_measured_csr(None, 2, 2, m, nnz) == 0
    assert lib.dgan_workspace_bytes_measured_csr(None, 2, 2, 10, 10) == 0       # no handle


def test_the_debug_layout_names_the_staged_csr():
    """The test aid exists (so the GPU tests can probe for the validation before passing malformed indices)."""
    from defensegan_b200 import _native
    lib = _native.load_library()
    fn = lib.dgan_debug_workspace_layout_measured_csr
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    buf = ctypes.create_string_buffer(1 << 12)
    assert fn(None, 4, 10, 10, buf, len(buf)) == -1


# ---- the binding ----

def _csr(m=50, seed=0):
    a = torch.tensor(SO.random_sparse_operator(m, 784, density=0.02, seed=seed))
    return a, a.to_sparse_csr()


def test_binding_passes_the_csr_through_unchanged(cpu_native):
    _, a = _csr()
    y = torch.rand(2, 50)
    nnz = a.values().numel()
    cpu_native.reconstruct_measured(y, a, 3, 5, 2.5, seed=11, momentum=0.5, decay_lr=True, out=cpu_native.Out(2 * 784),
                                    z_row_offset=6)
    rp, ci, val = cpu_native.seen["operator.crow_indices()"], cpu_native.seen["operator.col_indices()"], \
        cpu_native.seen["operator.values()"]
    assert rp.dtype == torch.int32 and ci.dtype == torch.int32                 # torch's int64 indices arrive as int32
    assert torch.equal(rp.long(), a.crow_indices()) and torch.equal(ci.long(), a.col_indices())
    assert torch.equal(val, a.values())
    cpu_native.loss_grad_measured(y, a, torch.zeros(6, 8), 3)
    calls = cpu_native.lib.calls
    assert [c[0] for c in calls] == ["dgan_workspace_bytes_measured_csr", "dgan_reconstruct_measured_csr",
                                     "dgan_workspace_bytes_measured_csr", "dgan_loss_grad_measured_csr"]
    assert calls[0][1][1:] == (2, 3, 50, nnz) and calls[2][1][1:] == (2, 3, 50, nnz)
    prm = calls[1][1][1]._obj
    assert (prm.batch, prm.rec_rr, prm.rec_iters, prm.rec_lr, prm.momentum, prm.decay_lr, prm.seed, prm.z_row_offset) == \
        (2, 3, 5, 2.5, 0.5, 1, 11, 6)
    args = calls[1][1]
    assert [p.value for p in args[2:5]] == [rp.data_ptr(), ci.data_ptr(), val.data_ptr()]
    assert args[5:7] == (50, nnz) and args[7].value == y.data_ptr()
    args = calls[3][1]
    assert args[4:6] == (50, nnz) and args[7:9] == (2, 3)


def test_binding_sends_a_strided_operator_to_the_dense_entry(cpu_native):
    a, _ = _csr()
    y = torch.rand(2, 50)
    cpu_native.reconstruct_measured(y, a, 3, 5, 2.5, out=cpu_native.Out(2 * 784))
    calls = cpu_native.lib.calls
    assert [c[0] for c in calls] == ["dgan_workspace_bytes_measured", "dgan_reconstruct_measured"]
    assert calls[0][1][1:] == (2, 3, 50)
    assert calls[1][1][2].value == a.data_ptr() and calls[1][1][3] == 50 and calls[1][1][4].value == y.data_ptr()


@pytest.mark.parametrize("shape,y_shape,match", [((50, 783), (2, 50), "operator"), ((785, 784), (2, 785), "operator"),
                                                 ((50, 784), (2, 49), "measurements")])
def test_binding_refuses_bad_csr_shapes(cpu_native, shape, y_shape, match):
    a = torch.zeros(shape)
    a[0, 0] = 1.0
    with pytest.raises(ValueError, match=match):
        cpu_native.reconstruct_measured(torch.rand(*y_shape), a.to_sparse_csr(), 3, 5)
    assert cpu_native.lib.calls == []


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


@pytest.mark.parametrize("layout", ["csr", "coo"])
def test_defensegan_passes_a_sparse_operator_as_csr(layout):
    gan, fake = _gan()
    gan.rec_rr, gan.rec_iters, gan.rec_lr = 4, 9, 3.0
    dense, a = _csr(30)
    if layout == "coo":
        a = dense.to_sparse()
        # an uncoalesced COO: the entries in reverse order, one of them split in two halves
        i, v = a.indices(), a.values()
        i = torch.cat([i.flip(1), i[:, :1]], dim=1)
        v = torch.cat([v.flip(0), torch.zeros(1)])
        v[-2] *= 0.5
        v[-1] = v[-2]
        a = torch.sparse_coo_tensor(i, v, dense.shape)
        assert not a.is_coalesced()
    y = np.random.RandomState(1).standard_normal((2, 30)).astype(np.float32)
    gan.reconstruct_measured(y, a, batch_size=2, z_row_offset=8)
    (yt, at, args, kw), = fake.calls
    assert at.layout == torch.sparse_csr and torch.equal(at.to_dense(), dense)
    assert torch.equal(yt, torch.as_tensor(y)) and args == (4, 9, 3.0)
    assert kw["z_row_offset"] == 8 and kw["momentum"] == float(gan.rec_momentum) and kw["seed"] == gan.last_seed


def _raw(crow, col, val, shape=(3, 784)):
    return torch.sparse_csr_tensor(torch.tensor(crow), torch.tensor(col), torch.tensor(val, dtype=torch.float32),
                                   size=shape, check_invariants=False)


def _batched():
    a = torch.eye(3, 784).to_sparse_csr()
    return torch.stack([a.to_dense(), a.to_dense()]).to_sparse_csr()


def _hybrid():
    return torch.ones(3, 784, 2).to_sparse_csr(dense_dim=1)


GOOD = ([0, 1, 1, 3], [5, 2, 700], [1.0, 2.0, 3.0])
BAD = {
    "wrong shape": (lambda: torch.eye(3, 783).to_sparse_csr(), "operator must be \\[m, 784\\]"),
    "batched": (_batched, "batched"),
    "hybrid": (_hybrid, "hybrid"),
    "column out of range": (lambda: _raw([0, 1, 1, 3], [5, 2, 784], [1.0, 2.0, 3.0]), "column indices must be in"),
    "negative column": (lambda: _raw([0, 1, 1, 3], [-1, 2, 7], [1.0, 2.0, 3.0]), "column indices must be in"),
    "unsorted columns": (lambda: _raw([0, 1, 1, 3], [5, 700, 2], [1.0, 2.0, 3.0]), "strictly ascending"),
    "duplicate columns": (lambda: _raw([0, 1, 1, 3], [5, 2, 2], [1.0, 2.0, 3.0]), "strictly ascending"),
    "decreasing crow_indices": (lambda: _raw([0, 2, 1, 3], [5, 2, 700], [1.0, 2.0, 3.0]), "crow_indices"),
    "crow_indices not from 0": (lambda: _raw([1, 1, 1, 3], [5, 2, 700], [1.0, 2.0, 3.0]), "crow_indices"),
    "crow_indices not to nnz": (lambda: _raw([0, 1, 1, 2], [5, 2, 700], [1.0, 2.0, 3.0]), "crow_indices"),
    "non-finite value": (lambda: _raw(GOOD[0], GOOD[1], [1.0, float("nan"), 3.0]), "operator values must be finite"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_malformed_csr_raises_before_any_native_call(case):
    make, match = BAD[case]
    gan, fake = _gan()
    counter = gan._call_counter
    with pytest.raises(ValueError, match=match):
        gan.reconstruct_measured(np.ones((2, 3), dtype=np.float32), make())
    assert fake.calls == [] and gan._call_counter == counter


def test_non_finite_measurements_raise_before_any_native_call():
    gan, fake = _gan()
    with pytest.raises(ValueError, match="^measurements must be finite"):
        gan.reconstruct_measured(np.full((2, 3), np.inf, dtype=np.float32), _raw(*GOOD))
    with pytest.raises(ValueError, match="measurements must be \\[B, 3\\]"):
        gan.reconstruct_measured(np.ones((2, 4), dtype=np.float32), _raw(*GOOD))
    assert fake.calls == []
    gan.reconstruct_measured(np.ones((2, 3), dtype=np.float32), _raw(*GOOD))       # the well-formed CSR passes
    assert len(fake.calls) == 1


def test_binding_refuses_an_nnz_int32_cannot_hold(cpu_native, monkeypatch):
    from defensegan_b200 import _native
    monkeypatch.setattr(_native, "INT32_MAX", 10)
    _, a = _csr()
    with pytest.raises(ValueError, match="non-zeros"):
        cpu_native.reconstruct_measured(torch.rand(2, 50), a, 3, 5)
    assert cpu_native.lib.calls == []


# ---- the test operators and the oracle ----

def test_operators():
    a = SO.blur_operator(6, 5, 3)
    assert a.shape == (90, 90) and ((a != 0).sum(axis=1) <= 25).all()
    np.testing.assert_allclose(a[(2 * 5 + 2) * 3 + 1].sum(), 1.0, rtol=1e-6)    # an interior row sums to 1
    x = np.random.RandomState(0).uniform(size=(6, 5, 3))
    k = np.exp(-0.5 * np.arange(-2, 3) ** 2)
    k /= k.sum()
    xp = np.pad(x, ((2, 2), (2, 2), (0, 0)))
    want = sum(k[i] * k[j] * xp[i:i + 6, j:j + 5] for i in range(5) for j in range(5))
    np.testing.assert_allclose(a @ x.reshape(-1), want.reshape(-1), rtol=1e-5)
    s = SO.subsample_operator(40, 784, seed=1)
    assert ((s != 0).sum(axis=1) == 1).all() and len(set(np.nonzero(s)[1])) == 40
    g = SO.grayscale_operator(4, 4)
    x = np.random.RandomState(0).uniform(size=(4, 4, 3))
    np.testing.assert_allclose(g @ x.reshape(-1), (x @ np.array([0.299, 0.587, 0.114])).reshape(-1), rtol=1e-5)
    r = SO.random_sparse_operator(20, 784, seed=2)
    assert not r[1].any() and (r[-1] != 0).all() and 0 < (r[0] != 0).sum() < 784


def test_oracle_is_the_same_for_an_operator_and_its_csr_densified():
    w = O.init_generator_weights("mnist", latent_dim=16, net_dim=8, random_bias=True)
    x = O.synthetic_images("mnist", w, 2, kind="S2", seed=3, latent_dim=16)
    z = O.sample_z0(4, 16, seed=3)
    a = SO.random_sparse_operator(30, 784, seed=4)
    back = torch.tensor(a).to_sparse_csr().to_dense().numpy()
    y = (x.reshape(2, -1) @ a.T).astype(np.float32)
    for p, q in zip(MO.loss_and_grad("mnist", w, a, y, z, 2), MO.loss_and_grad("mnist", w, back, y, z, 2)):
        assert np.array_equal(p, q)
