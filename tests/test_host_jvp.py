"""CPU tests of forward-mode differentiation of generator_fn: the forward-AD wiring of GeneratorFunction and the Jacobian
assembly, driven by a fake native generator, and the plans of the fp16 path's tangent directions (host code of the
CUDA library; no GPU)."""
import ctypes

import pytest
import torch
import torch.autograd.forward_ad as fwAD

from test_host_vjp import FakeNative
from test_host_widths import GRID, _desc


class FakeJvpNative(FakeNative):
    """FakeNative with jvp(z, t) = t @ A, the jacobian assembly of NativeGenerator and a use_bn switch."""

    def __init__(self, latent=4, out=6, use_bn=False):
        super().__init__(latent, out)
        self.latent_dim, self.use_bn = latent, use_bn
        self.image_dim = (out,)
        self.rows_per_call = []

    def jvp(self, z, t):
        z.data_ptr(), t.data_ptr()                   # the library reads storage: no functorch wrappers
        self.calls.append(("jvp", t.clone()))
        self.rows_per_call.append(t.shape[0])
        ty = torch.empty(t.shape[0], self.a.shape[1])   # and writes into buffers it was given
        ty.data_ptr()
        return ty.copy_(t @ self.a)

    def jacobian(self, z, max_rows=4096):
        from defensegan_b200 import _native
        return _native.NativeGenerator.jacobian(self, z, max_rows)


def _cpu_cuda_checks(monkeypatch):
    """NativeGenerator.jacobian validates its input as a CUDA tensor; on the CPU the fake takes any float tensor."""
    from defensegan_b200 import _native
    monkeypatch.setattr(_native, "_require_cuda_f32", lambda t, name: t.to(torch.float32).contiguous())


def test_forward_ad_calls_forward_then_jvp_with_the_tangent_unchanged():
    from defensegan_b200 import _native
    fake = FakeJvpNative()
    z, t = torch.randn(3, 4), torch.randn(3, 4)
    with fwAD.dual_level():
        y = _native.generator(fake, fwAD.make_dual(z, t))
        primal, tangent = fwAD.unpack_dual(y)
    assert torch.equal(primal, z @ fake.a)
    assert torch.equal(tangent, t @ fake.a)
    assert [c[0] for c in fake.calls] == ["forward", "jvp"]
    assert torch.equal(fake.calls[0][1], z) and torch.equal(fake.calls[1][1], t)


def test_torch_func_jvp_through_generator_fn():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    fake = FakeJvpNative(latent=128, out=5)
    gan._as_cuda = lambda t: t
    gan._get_native = lambda device: fake
    z, t = torch.randn(2, 128), torch.randn(2, 128)
    y, ty = torch.func.jvp(gan.generator_fn, (z,), (t,))
    assert torch.equal(y, z @ fake.a)
    assert torch.equal(ty, t @ fake.a)
    assert [c[0] for c in fake.calls] == ["forward", "jvp"]


def test_reverse_mode_logs_the_same_calls_as_before():
    from defensegan_b200 import _native
    fake = FakeJvpNative()
    z = torch.randn(3, 4, requires_grad=True)
    y = _native.generator(fake, z)
    dy = torch.randn(3, 6)
    y.backward(dy)
    assert [c[0] for c in fake.calls] == ["forward", "vjp"]
    assert torch.equal(z.grad, dy @ fake.a.t())
    y2 = _native.generator(fake, torch.randn(3, 4))
    assert y2.grad_fn is None and fwAD.unpack_dual(y2).tangent is None
    assert [c[0] for c in fake.calls] == ["forward", "vjp", "forward"]


@pytest.mark.parametrize("max_rows", [4096, 8, 9, 1])
def test_jacobian_assembly_matches_autograd(monkeypatch, max_rows):
    """[N, out, latent] from identity tangents, whole images per call, across chunk boundaries (8 rows = 2 images of 4
    latents; 9 rows still 2 images; 1 row: one image per call)."""
    _cpu_cuda_checks(monkeypatch)
    fake = FakeJvpNative()
    z = torch.randn(5, 4)
    got = fake.jacobian(z, max_rows=max_rows)
    want = torch.autograd.functional.jacobian(lambda zz: zz @ fake.a, z)     # [5, 6, 5, 4]
    want = torch.stack([want[i, :, i, :] for i in range(5)])
    assert got.shape == (5, 6, 4)
    assert torch.equal(got, want)
    per_call = max(1, max_rows // 4) * 4
    assert all(r % 4 == 0 and r <= per_call for r in fake.rows_per_call), fake.rows_per_call
    assert sum(fake.rows_per_call) == 5 * 4


def test_jacobian_refuses_batchnorm(monkeypatch):
    _cpu_cuda_checks(monkeypatch)
    fake = FakeJvpNative(use_bn=True)
    with pytest.raises(ValueError, match="BatchNorm"):
        fake.jacobian(torch.randn(2, 4))
    assert fake.calls == []


def test_generator_jacobian_delegates():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    seen = []

    class Native:
        def jacobian(self, z):
            seen.append(z)
            return "J"

    gan._as_cuda = lambda t: t
    gan._get_native = lambda device: Native()
    z = torch.randn(2, 128)
    assert gan.generator_jacobian(z) == "J" and seen[0] is z


def test_jvp_is_part_of_the_binding():
    from defensegan_b200 import _native
    assert "dgan_jvp" in _native.ABI_SYMBOLS
    assert callable(getattr(_native.NativeGenerator, "jvp"))
    assert callable(getattr(_native.NativeGenerator, "jacobian"))


# ---- plans of the tangent directions (dgan_debug_check_tangent_plans) ----

def _check_tangent(arch, latent, net_dim, use_bn, n_rows, n_pairs=66, mutate=0):
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_check_tangent_plans.restype = ctypes.c_int
    lib.dgan_debug_check_tangent_plans.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    d = _desc(arch, latent, net_dim, use_bn)
    rc = lib.dgan_debug_check_tangent_plans(ctypes.byref(d), n_rows, n_pairs, mutate)
    return rc, (lib.dgan_last_error() or b"").decode()


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", GRID + [("mnist", 128, 64, 0), ("celeba", 128, 64, 0),
                                                               ("mnist", 128, 64, 1)])
@pytest.mark.parametrize("n_rows", [1, 300, 2560])
def test_tangent_plans_pass_the_validator(arch, latent, net_dim, use_bn, n_rows):
    rc, msg = _check_tangent(arch, latent, net_dim, use_bn, n_rows)
    assert rc == 0, msg


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [("mnist", 128, 64, 0), ("celeba", 200, 48, 0), ("mnist", 128, 64, 1)])
def test_validator_names_the_damaged_tangent_direction(arch, latent, net_dim, use_bn):
    for mutate in range(1, 12):
        rc, msg = _check_tangent(arch, latent, net_dim, use_bn, 2560, mutate=mutate)
        assert rc != 0 and msg.startswith("Generator.3.jvp:"), (mutate, rc, msg)


def test_tangent_plans_for_random_widths_sizes_and_sm_counts():
    pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=40, deadline=None)
    @given(st.sampled_from(["mnist", "celeba"]), st.integers(1, 3000), st.integers(1, 74), st.integers(1, 256),
           st.integers(1, 128), st.sampled_from([0, 1]))
    def run(arch, n_rows, n_pairs, latent, net_dim, use_bn):
        rc, msg = _check_tangent(arch, latent, net_dim, use_bn, n_rows, n_pairs=n_pairs)
        assert rc == 0, (arch, n_rows, n_pairs, latent, net_dim, use_bn, msg)

    run()
