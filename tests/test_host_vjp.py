"""CPU tests of the autograd wiring of generator_fn: GeneratorFunction driven by a fake native generator."""
import pytest
import torch


class FakeNative:
    """Stands in for NativeGenerator: G(z) = z @ A, vjp(z, dy) = dy @ A^T, and a log of the calls."""

    def __init__(self, latent=4, out=6):
        self.a = torch.arange(latent * out, dtype=torch.float32).reshape(latent, out) / 10.0
        self.calls = []

    def forward(self, z):
        self.calls.append(("forward", z.detach().clone()))
        return z.detach() @ self.a

    def vjp(self, z, dy):
        self.calls.append(("vjp", dy.clone()))
        return dy @ self.a.t()


def test_backward_calls_vjp_once_with_the_cotangent_unchanged():
    from defensegan_b200 import _native
    fake = FakeNative()
    z = torch.randn(3, 4, requires_grad=True)
    y = _native.generator(fake, z)
    assert y.grad_fn is not None
    assert [c[0] for c in fake.calls] == ["forward"]
    assert torch.equal(fake.calls[0][1], z.detach())
    dy = torch.randn(3, 6)
    y.backward(dy)
    assert [c[0] for c in fake.calls] == ["forward", "vjp"]
    assert torch.equal(fake.calls[1][1], dy)
    assert torch.equal(z.grad, dy @ fake.a.t())
    with pytest.raises(RuntimeError):            # saved state is released by the first backward
        y.backward(dy)


def test_gradient_flows_through_a_user_loss():
    from defensegan_b200 import _native
    fake = FakeNative()
    z = torch.randn(2, 4, requires_grad=True)
    x = torch.randn(2, 6)
    ((_native.generator(fake, z) - x) ** 2).sum().backward()
    want = 2.0 * (z.detach() @ fake.a - x) @ fake.a.t()
    assert torch.allclose(z.grad, want)
    assert torch.equal(fake.calls[1][1], 2.0 * (z.detach() @ fake.a - x))


def test_without_grad_only_forward_runs():
    from defensegan_b200 import _native
    fake = FakeNative()
    y = _native.generator(fake, torch.randn(3, 4))
    assert y.grad_fn is None
    z = torch.randn(3, 4, requires_grad=True)
    with torch.no_grad():
        y2 = _native.generator(fake, z)
    assert y2.grad_fn is None and not y2.requires_grad
    assert [c[0] for c in fake.calls] == ["forward", "forward"]


def test_generator_fn_uses_the_autograd_function():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    fake = FakeNative(latent=128, out=5)
    gan._as_cuda = lambda t: t
    gan._get_native = lambda device: fake
    z = torch.randn(2, 128)
    assert gan.generator_fn(z).grad_fn is None
    z.requires_grad_(True)
    y = gan.generator_fn(z)
    y.sum().backward()
    assert [c[0] for c in fake.calls] == ["forward", "forward", "vjp"]
    assert torch.equal(z.grad, torch.ones(2, 5) @ fake.a.t())


def test_vjp_is_part_of_the_binding():
    from defensegan_b200 import _native
    assert "dgan_vjp" in _native.ABI_SYMBOLS
    assert callable(getattr(_native.NativeGenerator, "vjp"))
