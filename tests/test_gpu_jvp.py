"""Jacobian-vector products of the generator (dgan_jvp / NativeGenerator.jvp / generator_fn under forward-mode autograd /
NativeGenerator.jacobian) on an H100, against fp64 forward mode through the CPU oracle.

Tolerances (max |ty - ty64| / max |ty64|, cosine of ty and ty64):
  fp32: <= 2e-4, >= 0.999999  (as for the vector-Jacobian product)
  fp16: <= 1.5e-1, >= 0.998
The fp16 bound on the largest error is wider than the vjp's 6e-2.  Rounding in the fp16 forward flips the ReLU mask of
units whose pre-activation is ~0, in both modes.  A vjp's dz sums over every output pixel, so a flipped unit is a small
share of it.  Each pixel of J t depends on the few units under its 5x5 taps, so one flip can be a large share of that
pixel.  On an H100 the largest errors measured 4e-2 to 1.1e-1 over the configurations below, with cosines >= 0.9993.
The test shows the error comes from the primal forward, not from the tangent pass: at the pixel with the largest error,
J t computed in reverse mode, <J^T e_p, t> through dgan_vjp on the same fp16 forward, must agree with the jvp's value to
1e-2 of max |ty64|.
Adjoint identity with dgan_vjp, |<u, J t> - <J^T u, t>| / (|u| |J t|): fp32 <= 1e-5, fp16 <= 5e-2.
"""
import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16"]
TOL = {"fp32": dict(rel=2e-4, cos=0.999999, adj=1e-5), "fp16": dict(rel=1.5e-1, cos=0.998, adj=5e-2)}
# (arch, use_bn, rows, latent_dim, net_dim): the configurations of the vjp tests, then padded widths and column blocks
CONFIGS = [("mnist", False, 8, 128, 64), ("celeba", False, 4, 128, 64), ("mnist", True, 16, 128, 64),
           ("mnist", False, 6, 100, 32), ("celeba", False, 3, 200, 48), ("mnist", False, 5, 128, 128)]
CONFIG_IDS = ["mnist", "celeba", "mnist_bn", "mnist_l100_n32", "celeba_l200_n48", "mnist_n128"]


@pytest.fixture(scope="module")
def gens():
    from defensegan_b200 import _native
    cache = {}
    dev = torch.device("cuda", 0)

    def get(arch, use_bn, precision, latent=128, net_dim=64):
        key = (arch, use_bn, precision, latent, net_dim)
        if key not in cache:
            w = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, random_bias=True, use_bn=use_bn)
            cache[key] = (w, _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], latent_dim=latent,
                                                     net_dim=net_dim, use_bn=use_bn, precision=precision, device=dev))
        return cache[key]

    yield get
    for _, g in cache.values():
        g.close()


def _tangent(n, latent, kind, seed):
    rs = np.random.RandomState(seed)
    if kind == "dense":
        return rs.standard_normal((n, latent)).astype("float32")
    t = np.zeros((n, latent), "float32")          # one-hot: row i along latent direction k_i
    t[np.arange(n), rs.randint(0, latent, n)] = 1.0
    return t


def _oracle_jvp(arch, w, z, t, use_bn):
    w64 = O.weights_to_torch(w, torch.float64)
    _, ty = torch.func.jvp(lambda zz: O.generator_forward(arch, w64, zz, use_bn=use_bn),
                           (torch.tensor(z, dtype=torch.float64),), (torch.tensor(t, dtype=torch.float64),))
    return ty.numpy()


def _assert_close(got, want, precision, what):
    err = np.abs(got - want).max() / np.abs(want).max()
    cos = float((got * want).sum() / np.sqrt((got * got).sum() * (want * want).sum()))
    print("%s: rel %.2e cos %.8f" % (what, err, cos))
    assert err <= TOL[precision]["rel"], (what, err)
    assert cos >= TOL[precision]["cos"], (what, cos)


@pytest.mark.parametrize("kind", ["dense", "onehot"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg", CONFIGS, ids=CONFIG_IDS)
def test_jvp_matches_fp64_forward_mode_and_y_matches_forward(gens, cfg, precision, kind):
    arch, use_bn, n, latent, net_dim = cfg
    w, gen = gens(arch, use_bn, precision, latent, net_dim)
    z = O.sample_z0(n, latent, seed=11)
    t = _tangent(n, latent, kind, seed=12)
    zc, tc = torch.tensor(z).cuda(), torch.tensor(t).cuda()
    y, ty = gen.jvp(zc, tc, want_y=True)
    assert ty.shape == (n,) + gen.image_dim
    got, want = ty.cpu().numpy().astype(np.float64), _oracle_jvp(arch, w, z, t, use_bn)
    _assert_close(got, want, precision, "%s bn=%d l=%d n=%d %s %s" % (arch, use_bn, latent, net_dim, precision, kind))
    # the pixel with the largest error, in reverse mode on the same forward: <J^T e_p, t>
    p = np.unravel_index(np.abs(got - want).argmax(), got.shape)
    u = torch.zeros_like(ty)
    u[p] = 1.0
    rev = float((gen.vjp(zc, u).double() * tc.double()).sum())
    print("  worst pixel %s: jvp %.6f vjp %.6f fp64 %.6f" % (p, got[p], rev, want[p]))
    assert abs(rev - got[p]) <= 1e-2 * np.abs(want).max()
    assert torch.equal(y, gen.forward(zc))
    assert torch.equal(gen.jvp(zc, tc), ty)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg", CONFIGS[:3], ids=CONFIG_IDS[:3])
def test_jvp_is_exactly_homogeneous_in_t(gens, cfg, precision):
    """jvp(z, 2^k t) == 2^k jvp(z, t) bit for bit (the fp16 path's tangent scales are powers of two chosen from the data);
    without BatchNorm a row's result does not see the magnitude of another row's tangent."""
    arch, use_bn, n, latent, net_dim = cfg
    _, gen = gens(arch, use_bn, precision, latent, net_dim)
    z = torch.tensor(O.sample_z0(n, latent, seed=21)).cuda()
    t = torch.tensor(_tangent(n, latent, "dense", seed=22)).cuda()
    base = gen.jvp(z, t)
    assert bool(torch.isfinite(base).all()) and float(base.abs().max()) > 0
    for k in (-40, -12, 0, 12, 40):
        got = gen.jvp(z, t * 2.0 ** k)
        assert bool(torch.isfinite(got).all()), k
        assert torch.equal(got, base * 2.0 ** k), k
    if not use_bn:
        t2 = t.clone()
        t2[1:] *= 2.0 ** 30
        assert torch.equal(gen.jvp(z, t2)[0], base[0])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg", CONFIGS[:3], ids=CONFIG_IDS[:3])
def test_adjoint_identity_with_vjp(gens, cfg, precision):
    arch, use_bn, n, latent, net_dim = cfg
    _, gen = gens(arch, use_bn, precision, latent, net_dim)
    rs = np.random.RandomState(51)
    z = torch.tensor(O.sample_z0(n, latent, seed=50)).cuda()
    t = torch.tensor(rs.standard_normal((n, latent)).astype("float32")).cuda()
    u = torch.tensor(rs.standard_normal((n,) + gen.image_dim).astype("float32")).cuda()
    jt = gen.jvp(z, t).double()
    jtu = gen.vjp(z, u).double()
    lhs, rhs = float((u.double() * jt).sum()), float((jtu * t.double()).sum())
    gap = abs(lhs - rhs) / (float(u.double().norm()) * float(jt.norm()))
    print("%s bn=%d %s: <u, J t> %.6e  <J^T u, t> %.6e  gap %.2e" % (arch, use_bn, precision, lhs, rhs, gap))
    assert gap <= TOL[precision]["adj"], gap


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_mode_surface_of_generator_fn(precision):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision=precision)
    z = torch.tensor(O.sample_z0(5, 128, seed=31)).cuda()
    t = torch.tensor(_tangent(5, 128, "dense", seed=32)).cuda()
    native = gan._get_native(z.device)
    y_want, ty_want = native.jvp(z, t, want_y=True)
    # what the plain forward (the only path before generator_fn had a forward-mode rule) does with a tangent:
    # a dual tensor's tangent is dropped; a functorch-wrapped tensor has no storage to hand to the library
    with fwAD.dual_level():
        assert fwAD.unpack_dual(native.forward(fwAD.make_dual(z, t))).tangent is None
    try:
        _, ty_plain = torch.func.jvp(native.forward, (z,), (t,))
        outcome = "tangent lost" if not bool(ty_plain.any()) else "tangent kept"
    except RuntimeError as e:
        outcome = "error: %s" % str(e).splitlines()[0]
    print("torch.func.jvp through the plain forward:", outcome)
    assert outcome != "tangent kept"
    with fwAD.dual_level():
        primal, tangent = fwAD.unpack_dual(gan.generator_fn(fwAD.make_dual(z, t)))
    assert torch.equal(primal, y_want) and torch.equal(tangent, ty_want)
    y, ty = torch.func.jvp(gan.generator_fn, (z,), (t,))
    assert torch.equal(y, y_want) and torch.equal(ty, ty_want)
    assert torch.equal(gan.generator_fn(z), y_want)
    with pytest.raises(ValueError):
        native.jvp(z, t[:, :64])
    with pytest.raises(ValueError):
        native.jvp(z, t[:4])
    gan.close()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_generator_jacobian(gens, arch, precision):
    """Against torch.autograd.functional.jacobian of the fp64 oracle for 2 images; column k is jvp(z, e_k) bit for bit,
    and one image per call gives the same bits as all images in one call."""
    from defensegan_b200.models.gan import CelebADefenseGAN, MnistDefenseGAN
    w, gen = gens(arch, False, precision)
    z = O.sample_z0(3, 128, seed=61)
    zc = torch.tensor(z).cuda()
    jac = gen.jacobian(zc)
    assert jac.shape == (3,) + gen.image_dim + (128,)
    w64 = O.weights_to_torch(w, torch.float64)
    for i in range(2):
        want = torch.autograd.functional.jacobian(lambda zz: O.generator_forward(arch, w64, zz[None])[0],
                                                  torch.tensor(z[i], dtype=torch.float64), vectorize=True,
                                                  strategy="forward-mode")
        _assert_close(jac[i].cpu().numpy().astype(np.float64), want.numpy(), precision, "%s %s J[%d]" % (arch, precision, i))
    for k in (0, 1, 77, 127):
        e = torch.zeros(3, 128, device="cuda")
        e[:, k] = 1.0
        assert torch.equal(jac[..., k], gen.jvp(zc, e)), k
    assert torch.equal(gen.jacobian(zc, max_rows=128), jac)
    gan = (MnistDefenseGAN if arch == "mnist" else CelebADefenseGAN)(test_mode=True, verbose=False, precision=precision)
    gan.weights = w
    assert torch.equal(gan.generator_jacobian(zc), jac)
    gan.close()
    _, gen_bn = gens("mnist", True, precision)
    with pytest.raises(ValueError, match="BatchNorm"):
        gen_bn.jacobian(zc)


def test_jvp_does_not_allocate_at_a_planned_size(gens):
    for precision in PRECISIONS:
        _, gen = gens("mnist", False, precision)
        z = torch.tensor(O.sample_z0(12, 128, seed=41)).cuda()
        t = torch.tensor(_tangent(12, 128, "dense", seed=42)).cuda()
        want = gen.jvp(z, t).clone()                  # plans the tangent pass for 12 rows
        assert torch.equal(gen.jvp(z, t), want)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for _ in range(3):
            assert torch.equal(gen.jvp(z, t), want)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_jvp_leaves_the_projection_unchanged(gens, precision):
    """On one handle, a reconstruct before and after a jvp (at the projection's row count and at another) gives the same
    bits and runs the same launches."""
    w, gen = gens("mnist", False, precision)
    B, R, L = 4, 3, 20
    x = torch.tensor(O.synthetic_images("mnist", w, B, kind="S2", seed=5)).cuda()

    def run():
        rec, loss, idx = gen.reconstruct(x, R, L, seed=7, return_aux=True)
        torch.cuda.synchronize()
        return rec.clone(), loss.clone(), idx.clone(), gen.last_launch_count, gen.last_enqueue_count

    before = run()
    for n in (B * R, 40):
        gen.jvp(torch.tensor(O.sample_z0(n, 128, seed=n)).cuda(), torch.tensor(_tangent(n, 128, "dense", seed=n)).cuda())
    after = run()
    for a, b in zip(before[:3], after[:3]):
        assert torch.equal(a, b)
    assert before[3:] == after[3:]
