"""CPU tests (no GPU) of the projection from linear measurements: the measured oracle against the existing oracles and
the binding's and DefenseGANBase's argument handling."""
import ctypes
import os

import numpy as np
import pytest
import torch

import measured_oracle as MO
import weighted_oracle as WO
from oracle import defensegan_oracle as O

from recording import Out, cpu_native  # noqa: F401  (the fixture)


def _problem(arch="mnist", b=2, rr=2, latent=16, net_dim=8, seed=3):
    w = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, random_bias=True)
    x = O.synthetic_images(arch, w, b, kind="S2", seed=seed, latent_dim=latent)
    z = O.sample_z0(b * rr, latent, seed=seed)
    return w, x, z


# ---- the measured oracle ----

@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_oracle_identity_operator_is_reconstruct(arch):
    w, x, z = _problem(arch)
    hwc = x[0].size
    eye = np.eye(hwc, dtype=np.float64)
    y = x.reshape(x.shape[0], -1).astype(np.float64)
    for a, b in zip(MO.loss_and_grad(arch, w, eye, y, z, 2, dtype=torch.float64),
                    O.loss_and_grad(arch, w, x, z, 2, dtype=torch.float64)):
        np.testing.assert_allclose(a.reshape(b.shape), b, rtol=1e-12, atol=1e-15)
    got = MO.reconstruct(arch, w, eye, y, 2, 3, z_init_val=z, dtype=torch.float64)
    want = O.reconstruct(arch, w, x, 2, 3, z_init_val=z, dtype=torch.float64)
    for k in ("loss_min", "loss_all", "z_final"):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-10, atol=1e-14, err_msg=k)
    np.testing.assert_allclose(got["rec"], want["rec"], rtol=1e-10, atol=1e-14)
    assert np.array_equal(got["idx"], want["idx"])


def test_oracle_diagonal_operator_is_the_weighted_oracle():
    w, x, z = _problem()
    pw = np.random.RandomState(1).uniform(0, 1, size=x.shape)
    s = np.sqrt(pw.reshape(x.shape[0], -1)[0])
    pw = np.ascontiguousarray(np.broadcast_to(s.reshape(x.shape[1:]) ** 2, x.shape))
    a = np.diag(s)
    y = x.reshape(x.shape[0], -1).astype(np.float64) * s
    for p, q in zip(MO.loss_and_grad("mnist", w, a, y, z, 2, dtype=torch.float64),
                    WO.loss_and_grad("mnist", w, x, z, 2, dtype=torch.float64, pixel_weights=pw)):
        np.testing.assert_allclose(p.reshape(q.shape), q, rtol=1e-10, atol=1e-14)
    got = MO.reconstruct("mnist", w, a, y, 2, 3, z_init_val=z, dtype=torch.float64)
    want = WO.reconstruct("mnist", w, x, 2, 3, z_init_val=z, dtype=torch.float64, pixel_weights=pw)
    for k in ("loss_min", "loss_all", "z_final"):
        np.testing.assert_allclose(got[k], want[k], rtol=1e-9, atol=1e-14, err_msg=k)
    assert np.array_equal(got["idx"], want["idx"])


@pytest.mark.parametrize("m", [1, 37])
def test_oracle_gradient_is_autograd_of_the_measured_loss(m):
    w, x, z = _problem(b=2, rr=2, latent=8)
    a = MO.gaussian_operator(m, 784, seed=2).astype(np.float64)
    y = x.reshape(2, -1).astype(np.float64) @ a.T + 0.1
    _, loss, g = MO.loss_and_grad("mnist", w, a, y, z, 2, dtype=torch.float64)
    # the definition, written out: (1/m) ||A G(z) - y[n // R]||^2 per row
    wt = O.weights_to_torch(w, torch.float64)
    zt = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    gz = O.generator_forward("mnist", wt, zt).reshape(4, -1)
    r = gz @ torch.tensor(a).t() - torch.tensor(y)[[0, 0, 1, 1]]
    want = (r ** 2).sum(dim=1) / m
    (gw,) = torch.autograd.grad(want.sum(), zt)
    np.testing.assert_allclose(loss, want.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(g, gw.numpy(), rtol=1e-10, atol=1e-14)


def test_block_average_operator():
    a = MO.block_average_operator(4, 4, 3, 2)
    x = np.random.RandomState(0).uniform(size=(4, 4, 3))
    want = x.reshape(2, 2, 2, 2, 3).mean(axis=(1, 3)).reshape(-1)
    np.testing.assert_allclose(a @ x.reshape(-1), want, rtol=1e-6)


# ---- the C-ABI and the binding ----

def test_workspace_bytes_measured_refuses_bad_m_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    for m in (0, -1, 785):
        assert lib.dgan_workspace_bytes_measured(None, 2, 2, m) == 0


def test_binding_passes_the_arguments_unchanged(cpu_native):
    a, y = torch.rand(50, 784), torch.rand(2, 50)
    cpu_native.reconstruct_measured(y, a, 3, 5, 2.5, seed=11, momentum=0.5, decay_lr=True, out=cpu_native.Out(2 * 784),
                                    z_row_offset=6)
    cpu_native.loss_grad_measured(y, a, torch.zeros(6, 8), 3)
    calls = cpu_native.lib.calls
    assert [c[0] for c in calls] == ["dgan_workspace_bytes_measured", "dgan_reconstruct_measured",
                                     "dgan_workspace_bytes_measured", "dgan_loss_grad_measured"]
    assert calls[0][1][1:] == (2, 3, 50) and calls[2][1][1:] == (2, 3, 50)
    prm = calls[1][1][1]._obj
    assert (prm.batch, prm.rec_rr, prm.rec_iters, prm.rec_lr, prm.momentum, prm.decay_lr, prm.seed, prm.z_row_offset) == \
        (2, 3, 5, 2.5, 0.5, 1, 11, 6)
    assert calls[1][1][2].value == a.data_ptr() and calls[1][1][3] == 50 and calls[1][1][4].value == y.data_ptr()
    assert calls[3][1][1].value == a.data_ptr() and calls[3][1][2:6] == (50, calls[3][1][3], 2, 3)


@pytest.mark.parametrize("a_shape,y_shape,match", [((50, 783), (2, 50), "operator"), ((785, 784), (2, 785), "operator"),
                                                   ((0, 784), (2, 0), "operator"), ((50, 784), (2, 49), "measurements"),
                                                   ((50, 784), (50,), "measurements")])
def test_binding_refuses_bad_shapes(cpu_native, a_shape, y_shape, match):
    with pytest.raises(ValueError, match=match):
        cpu_native.reconstruct_measured(torch.rand(*y_shape), torch.rand(*a_shape), 3, 5)
    assert cpu_native.lib.calls == []


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
    gan._as_cuda = lambda t: torch.as_tensor(t).to(torch.float32)
    gan._get_native = lambda device: fake
    return gan, fake


def test_defensegan_passes_numpy_inputs_and_its_hyper_parameters():
    gan, fake = _gan()
    gan.rec_rr, gan.rec_iters, gan.rec_lr = 4, 9, 3.0
    a = np.random.RandomState(0).standard_normal((30, 784)).astype(np.float32)
    y = np.random.RandomState(1).standard_normal((2, 30)).astype(np.float32)
    gan.reconstruct_measured(y, a, batch_size=2, z_row_offset=8)
    (yt, at, args, kw), = fake.calls
    assert torch.equal(yt, torch.as_tensor(y)) and torch.equal(at, torch.as_tensor(a)) and args == (4, 9, 3.0)
    assert kw["z_row_offset"] == 8 and kw["momentum"] == float(gan.rec_momentum) and kw["seed"] == gan.last_seed


@pytest.mark.parametrize("a,y,kw,match", [
    (np.ones((30, 783)), np.ones((2, 30)), {}, "operator"),
    (np.ones((785, 784)), np.ones((2, 785)), {}, "operator"),
    (np.ones((30, 784)), np.ones((2, 31)), {}, "measurements"),
    (np.ones((30, 784)), np.ones((2, 30)), {"batch_size": 3}, "batch_size"),
    (np.full((30, 784), np.nan), np.ones((2, 30)), {}, "operator must be finite"),
    (np.ones((30, 784)), np.full((2, 30), np.inf), {}, "^measurements must be finite"),
])
def test_bad_inputs_raise_before_any_native_call(a, y, kw, match):
    gan, fake = _gan()
    counter = gan._call_counter
    with pytest.raises(ValueError, match=match):
        gan.reconstruct_measured(y, a, **kw)
    assert fake.calls == [] and gan._call_counter == counter
