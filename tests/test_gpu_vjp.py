"""Vector-Jacobian products of the generator (dgan_vjp / NativeGenerator.vjp / generator_fn under autograd) on an H100,
against fp64 autograd through the CPU oracle.

Tolerances, as for the projection's gradient (max |dz - dz64| / max |dz64|, cosine of dz and dz64):
  fp32: <= 2e-4, >= 0.999999
  fp16: <= 6e-2, >= 0.998   (rounding flips the ReLU mask of units whose pre-activation is ~0)
"""
import os

import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16"]
TOL = {
    "fp32": dict(grad_rel=2e-4, grad_cos=0.999999, rec=1e-4),
    "fp16": dict(grad_rel=6e-2, grad_cos=0.998, rec=2e-2),
}
# (arch, use_bn, rows)
CONFIGS = [("mnist", False, 8), ("celeba", False, 4), ("mnist", True, 16)]
CONFIG_IDS = ["mnist", "celeba", "mnist_bn"]


@pytest.fixture(scope="module")
def gens():
    from defensegan_b200 import _native
    cache = {}
    dev = torch.device("cuda", 0)

    def get(arch, use_bn, precision):
        key = (arch, use_bn, precision)
        if key not in cache:
            w = O.init_generator_weights(arch, random_bias=True, use_bn=use_bn)
            cache[key] = (w, _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()],
                                                     use_bn=use_bn, precision=precision, device=dev))
        return cache[key]

    yield get
    for _, g in cache.values():
        g.close()


def _cotangent(shape, kind, seed):
    rs = np.random.RandomState(seed)
    dy = rs.standard_normal(shape).astype("float32")
    if kind == "sparse":                               # non-zero on ~1 % of the pixels (all channels of a pixel)
        dy *= (rs.rand(*shape[:3], 1) < 0.01).astype("float32")
        dy[:, 0, 0, :] = rs.standard_normal((shape[0], shape[3]))   # and on at least one pixel per row
    return dy


def _oracle_vjp(arch, w, z, dy, use_bn):
    zt = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    y = O.generator_forward(arch, O.weights_to_torch(w, torch.float64), zt, use_bn=use_bn)
    (g,) = torch.autograd.grad(y, zt, torch.tensor(dy, dtype=torch.float64))
    return g.numpy()


def _assert_close_grad(got, want, precision, what):
    t = TOL[precision]
    err = np.abs(got - want).max() / np.abs(want).max()
    cos = float((got * want).sum() / np.sqrt((got * got).sum() * (want * want).sum()))
    print("%s: rel %.2e cos %.8f" % (what, err, cos))
    assert err <= t["grad_rel"], (what, err)
    assert cos >= t["grad_cos"], (what, cos)


@pytest.mark.parametrize("kind", ["dense", "sparse"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg", CONFIGS, ids=CONFIG_IDS)
def test_vjp_matches_fp64_autograd_and_y_matches_forward(gens, cfg, precision, kind):
    arch, use_bn, n = cfg
    w, gen = gens(arch, use_bn, precision)
    z = O.sample_z0(n, 128, seed=11)
    dy = _cotangent((n,) + gen.image_dim, kind, seed=12)
    y, dz = gen.vjp(torch.tensor(z).cuda(), torch.tensor(dy).cuda(), want_y=True)
    _assert_close_grad(dz.cpu().numpy().astype(np.float64), _oracle_vjp(arch, w, z, dy, use_bn), precision,
                       "%s bn=%d %s %s" % (arch, use_bn, precision, kind))
    assert torch.equal(y, gen.forward(torch.tensor(z).cuda()))
    assert torch.equal(gen.vjp(torch.tensor(z).cuda(), torch.tensor(dy).cuda()), dz)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg", CONFIGS, ids=CONFIG_IDS)
def test_vjp_is_exactly_homogeneous_in_dy(gens, cfg, precision):
    """vjp(z, 2^k dy) == 2^k vjp(z, dy) bit for bit (the fp16 path's cotangent scales are powers of two chosen from the
    data); without BatchNorm a row's result does not see the magnitude of another row's cotangent."""
    arch, use_bn, n = cfg
    _, gen = gens(arch, use_bn, precision)
    z = torch.tensor(O.sample_z0(n, 128, seed=21)).cuda()
    dy = torch.tensor(_cotangent((n,) + gen.image_dim, "dense", seed=22)).cuda()
    base = gen.vjp(z, dy)
    assert bool(torch.isfinite(base).all()) and float(base.abs().max()) > 0
    for k in (-40, -12, 0, 12, 40):
        got = gen.vjp(z, dy * 2.0 ** k)
        assert bool(torch.isfinite(got).all()), k
        assert torch.equal(got, base * 2.0 ** k), k
    if not use_bn:
        dy2 = dy.clone()
        dy2[1:] *= 2.0 ** 30
        assert torch.equal(gen.vjp(z, dy2)[0], base[0])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_vjp_of_the_projection_cotangent_matches_loss_grad(gens, arch, precision):
    w, gen = gens(arch, False, precision)
    B, R = 3, 2
    x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=5)).cuda()
    z = torch.tensor(O.sample_z0(B * R, 128, seed=6)).cuda()
    y = gen.forward(z)
    dy = 2.0 * (y - O.tile_images(x, R)) / gen.hwc
    _, _, grad = gen.loss_grad(x, z, R)
    _assert_close_grad(gen.vjp(z, dy).cpu().numpy().astype(np.float64), grad.cpu().numpy().astype(np.float64), precision,
                       "%s %s vs loss_grad" % (arch, precision))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", ["mnist_c1", "celeba_small"])
def test_projection_through_autograd_matches_golden(golden_dir, case, precision):
    """The projection written by a user: torch.optim.SGD(momentum=0.7) on z through generator_fn for L-1 steps, then
    G(z) and the per-image arg-min, against the fp64 oracle's reconstruction."""
    from defensegan_b200.models.gan import CelebADefenseGAN, MnistDefenseGAN
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    arch, B, R, L, lr = str(g["arch"]), int(g["B"]), int(g["R"]), int(g["L"]), float(g["lr"])
    gan = (MnistDefenseGAN if arch == "mnist" else CelebADefenseGAN)(test_mode=True, verbose=False, precision=precision,
                                                                       use_bn=False)
    gan.set_generator_weights(O.init_generator_weights(arch, random_bias=bool(int(g["random_bias"]))))
    x_tiled = O.tile_images(torch.tensor(g["images"]).cuda(), R)
    z = torch.tensor(g["z0"]).cuda().requires_grad_(True)
    opt = torch.optim.SGD([z], lr=lr, momentum=0.7)
    for _ in range(L - 1):
        opt.zero_grad()
        ((gan.generator_fn(z) - x_tiled) ** 2).mean(dim=(1, 2, 3)).sum().backward()
        opt.step()
    with torch.no_grad():
        y = gan.generator_fn(z)
        loss = ((y - x_tiled) ** 2).mean(dim=(1, 2, 3)).view(B, R)
        idx = loss.argmin(dim=1)
        rec = y.view(B, R, *y.shape[1:])[torch.arange(B, device=y.device), idx]
    np.testing.assert_array_equal(idx.cpu().numpy(), g["idx64"])
    err = np.abs(rec.cpu().numpy() - g["rec64"]).max()
    print("%s %s: max|rec - rec64| = %.2e" % (case, precision, err))
    assert err <= TOL[precision]["rec"]
    gan.close()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_generator_fn_autograd_surface(precision):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision=precision)
    z0 = torch.tensor(O.sample_z0(5, 128, seed=31)).cuda()
    native = gan._get_native(z0.device)
    want = native.forward(z0)
    y = gan.generator_fn(z0)
    assert y.grad_fn is None and not y.requires_grad and torch.equal(y, want)
    z = z0.clone().requires_grad_(True)
    with torch.no_grad():
        y = gan.generator_fn(z)
    assert y.grad_fn is None and torch.equal(y, want)
    y = gan.generator_fn(z)
    assert y.grad_fn is not None and torch.equal(y.detach(), want)
    dy = torch.tensor(_cotangent((5, 28, 28, 1), "dense", seed=32)).cuda()
    y.backward(dy)
    assert torch.equal(z.grad, native.vjp(z0, dy))
    with pytest.raises(RuntimeError):
        y.backward(dy)
    with pytest.raises(ValueError):
        native.vjp(z0, dy[:, :14])
    with pytest.raises(ValueError):
        native.vjp(z0, dy[:4])
    gan.close()


def test_vjp_does_not_allocate_at_a_planned_size(gens):
    for precision in PRECISIONS:
        _, gen = gens("mnist", False, precision)
        z = torch.tensor(O.sample_z0(12, 128, seed=41)).cuda()
        dy = torch.tensor(_cotangent((12, 28, 28, 1), "dense", seed=42)).cuda()
        want = gen.vjp(z, dy).clone()
        assert torch.equal(gen.vjp(z, dy), want)      # (also warms torch's own allocator)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for _ in range(3):
            assert torch.equal(gen.vjp(z, dy), want)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
