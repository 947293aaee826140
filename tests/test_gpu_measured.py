"""GPU tests (H100, -m gpu) of the projection from linear measurements (dgan_reconstruct_measured,
dgan_loss_grad_measured), on both precisions, MNIST and CelebA:
  - A = I with y = x gives reconstruct's outputs, and A = diag(sqrt(w)) with y = sqrt(w) x gives the weighted call's,
    within test_gpu_weighted.py's tolerances (with and without BatchNorm);
  - R = 10, L = 200 against the measured CPU oracle (tests/measured_oracle.py) within test_gpu_parity.py's long-horizon
    bar, for Gaussian sketches whose m is no multiple of any tile and a 2x2 block average; one loss / gradient evaluation
    against its fp64 evaluation;
  - both measurement products against fp64 on the operands they read, read back from the workspace;
  - isolation: one image's measurements do not change a bit of another's outputs, and a zero row appended to A (with a
    zero appended to y) changes nothing beyond rounding;
  - steady state: no allocation, the captured loop replayed, the documented launch and enqueue counts, and measured,
    plain and weighted calls alternating on one workspace give the bits of fresh calls."""
import ctypes

import numpy as np
import pytest
import torch

import measured_oracle as MO
from gpu_support import HWC, SHAPE, TOL, check_products, layout, release_cached_memory, views  # noqa: F401
from gpu_support import gen as _gen
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


def _measure(a, x):
    """y = A x for images x [B, H, W, C] (torch, on the GPU), in fp64."""
    return (x.reshape(x.shape[0], -1).double() @ a.double().t()).float()


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_identity_operator_gives_reconstruct(precision, arch, use_bn):
    w, gen = _gen(arch, precision, use_bn)
    try:
        # with BatchNorm the loop runs at the step of the BN golden cases (test_gpu_parity.py): the batch statistics of six
        # rows couple every row's rounding into every row, and L steps of lr 10 amplify it beyond any fixed tolerance
        B, R_, L, lr = (3, 2, 3, 0.5) if use_bn else (3, 2, 6, 10.0)
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        eye = torch.eye(HWC[arch], device="cuda")
        t = TOL[precision]
        # one loop body at z0
        y, l1, g1 = gen.loss_grad(x, z0, R_)
        my, ml1, mg1 = gen.loss_grad_measured(x.reshape(B, -1), eye, z0, R_)
        assert torch.equal(my, y)
        assert float((ml1 - l1).abs().max()) <= t["loss"]
        assert float((mg1 - g1).abs().max() / g1.abs().max()) <= t["grad_rel"]
        rec, loss, idx = gen.reconstruct(x, R_, L, lr, z_init_val=z0, return_aux=True)
        mrec, mloss, midx = gen.reconstruct_measured(x.reshape(B, -1), eye, R_, L, lr, z_init_val=z0, return_aux=True)
        if use_bn:     # the loop's tolerances of test_gpu_parity.py's BN test (fp16: pixels move by a few 1e-2)
            rt, lt = {"fp32": (1e-3, 1e-4), "fp16": (1e-1, 1e-3)}[precision]
        else:
            rt, lt = t["fwd"], t["loss"]
        print("\n%s %s bn=%d: |drec| %.3g |dloss| %.3g" % (precision, arch, use_bn, float((mrec - rec).abs().max()),
                                                       float((mloss - loss).abs().max())))
        assert float((mrec - rec).abs().max()) <= rt
        assert float((mloss - loss).abs().max()) <= lt
        assert torch.equal(midx, idx) if precision == "fp32" or not use_bn else float((midx == idx).float().mean()) >= 0.5
        # the same seed starts from the same z0
        a = gen.reconstruct(x, R_, 1, 10.0, seed=7)
        b = gen.reconstruct_measured(x.reshape(B, -1), eye, R_, 1, 10.0, seed=7)
        assert float((a - b).abs().max()) <= t["fwd"]
    finally:
        gen.close()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_diagonal_operator_gives_the_weighted_reconstruct(precision, arch):
    w, gen = _gen(arch, precision)
    try:
        B, R_, L = 3, 2, 6
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        pw = torch.rand(SHAPE[arch], generator=torch.Generator().manual_seed(5)).cuda()
        s = pw.reshape(-1).sqrt()
        t = TOL[precision]
        rec, loss, idx = gen.reconstruct(x, R_, L, 10.0, z_init_val=z0, return_aux=True,
                                         pixel_weights=pw.expand_as(x).contiguous())
        mrec, mloss, midx = gen.reconstruct_measured(x.reshape(B, -1) * s, torch.diag(s), R_, L, 10.0, z_init_val=z0,
                                                     return_aux=True)
        assert float((mrec - rec).abs().max()) <= t["fwd"]
        assert float((mloss - loss).abs().max()) <= t["loss"]
        assert torch.equal(midx, idx)
    finally:
        gen.close()


def _operator(arch, kind):
    h, w_, c = SHAPE[arch]
    if kind == "block2":
        return MO.block_average_operator(h, w_, c, 2)
    return MO.gaussian_operator(int(kind[5:]), HWC[arch], seed=int(kind[5:]))


def _lr(a):
    """rec_lr for operator a: the step of reconstruct's on the measured subspace (rows of about unit norm give gradients
    about H*W*C / m times reconstruct's; the block average's rows give its gradient exactly)."""
    m, hwc = a.shape
    return 10.0 if m * 4 == hwc else 10.0 * m / hwc


_ORACLE = {}
LONG = [("mnist", "gauss1"), ("mnist", "gauss50"), ("mnist", "gauss200"), ("mnist", "block2"),
        ("celeba", "gauss100"), ("celeba", "gauss1000"), ("celeba", "block2")]


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,kind", LONG)
def test_long_horizon_measured_parity(arch, kind, precision):
    """R = 10, L = 200: per-image |loss_min - oracle| <= 1e-4, the bar of test_gpu_parity.py's long-horizon test, on the
    measured loss; the returned loss is the measured loss of the returned reconstruction."""
    B, R_, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    w, gen = _gen(arch, precision)
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R_, 128)
        a = _operator(arch, kind)
        y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        if (arch, kind) not in _ORACLE:
            _ORACLE[(arch, kind)] = MO.reconstruct(arch, w, a, y, R_, L, rec_lr=_lr(a), z_init_val=z0)
        ref = _ORACLE[(arch, kind)]
        at = torch.tensor(a).cuda()
        rec, loss, idx = gen.reconstruct_measured(torch.tensor(y).cuda(), at, R_, L, _lr(a), z_init_val=torch.tensor(z0).cuda(),
                                                  return_aux=True)
        dl = np.abs(loss.cpu().numpy() - ref["loss_min"])
        agree = float((idx.cpu().numpy() == ref["idx"]).mean())
        print("%s %s m=%d %s: max|dloss|=%.3g (loss %.3g) restart agreement=%.2f"
              % (precision, arch, a.shape[0], kind, dl.max(), float(ref["loss_min"].max()), agree))
        assert dl.max() <= 1e-4
        ml = ((rec.reshape(B, -1).double() @ at.double().t() - torch.tensor(y).cuda().double()) ** 2).mean(dim=1)
        # fp16 path: the loss is that of the TF32 measurement product
        tol = 1e-5 if precision == "fp32" else TOL["fp16"]["loss"]
        assert float((ml - loss.double()).abs().max()) <= tol * max(1.0, float(ml.abs().max()))
    finally:
        gen.close()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_measured_loss_and_grad_match_fp64_oracle(precision, arch):
    w, gen = _gen(arch, precision)
    try:
        B, R_ = 3, 2
        imgs = O.synthetic_images(arch, w, B, kind="S2", seed=5)
        z = O.sample_z0(B * R_, 128, seed=6)
        a = MO.gaussian_operator(200 if arch == "mnist" else 1000, HWC[arch], seed=3)
        y = (imgs.reshape(B, -1) @ a.T).astype(np.float32)
        g64, loss64, grad64 = MO.loss_and_grad(arch, w, a, y, z, R_, dtype=torch.float64)
        g, loss, grad = gen.loss_grad_measured(torch.tensor(y).cuda(), torch.tensor(a).cuda(), torch.tensor(z).cuda(), R_)
        t = TOL[precision]
        assert np.abs(g.cpu().numpy() - g64).max() <= t["fwd"]
        assert np.abs(loss.cpu().numpy() - loss64).max() <= t["loss"] * max(1.0, float(np.abs(loss64).max()))
        gr = grad.cpu().numpy()
        assert np.abs(gr - grad64).max() / np.abs(grad64).max() <= t["grad_rel"]
        assert float((gr * grad64).sum() / np.sqrt((gr * gr).sum() * (grad64 * grad64).sum())) >= t["grad_cos"]
    finally:
        gen.close()


@pytest.mark.parametrize("m", [1, 50, 200, 784])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_each_measurement_product_on_its_stored_operands(arch, precision, m):
    """r = A G - y and dy = (2/m) A^T r against fp64 on the operands the kernels read (G in "y", A in "am", A^T in "amt",
    y in "ym", r in "r"), each within the bound of its arithmetic: fp32 accumulation of K terms, gamma_K = K u / (1 - K u)
    with u = 2^-24, times sum |terms|; on the fp16 path the operands are rounded to TF32 first (relative 2^-11 each)."""
    w, gen = _gen(arch, precision)
    try:
        B, R_ = 150, 2
        hwc = HWC[arch]
        n = B * R_
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, hwc, seed=m)).cuda()
        y = _measure(a, imgs) + 0.01 * torch.randn(B, m, generator=torch.Generator().manual_seed(1)).cuda()
        z = torch.tensor(O.sample_z0(n, 128, seed=4)).cuda()
        gen.loss_grad_measured(y, a, z, R_)
        torch.cuda.synchronize()
        ws = views(gen, layout(gen, "_measured", n, m)[0][0])
        m_ld = ws["am"].shape[0]
        assert m_ld % 64 == 0 and m_ld >= m
        assert torch.equal(ws["am"][:m], a) and not ws["am"][m:].any()
        assert torch.equal(ws["amt"], ws["am"].t()) and torch.equal(ws["ym"][:B, :m], y) and not ws["ym"][:B, m:].any()
        r_ratio, dy_ratio = check_products(ws, n, R_, m, hwc, precision)
        print("\n%s %s m=%d: r max err / bound %.3g" % (precision, arch, m, r_ratio))
        print("%s %s m=%d: dy max err / bound %.3g" % (precision, arch, m, dy_ratio))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_images_are_isolated_and_padding_is_never_observed(precision):
    arch, B, R_, L, m = "mnist", 4, 3, 8, 64
    w, gen = _gen(arch, precision)
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, 784, seed=9)).cuda()
        y = _measure(a, x)
        lr = 10.0 * m / 784
        base = gen.reconstruct_measured(y, a, R_, L, lr, z_init_val=z0, return_aux=True)
        y2 = y.clone()
        y2[2] = torch.randn(m, generator=torch.Generator().manual_seed(3)).cuda()
        other = gen.reconstruct_measured(y2, a, R_, L, lr, z_init_val=z0, return_aux=True)
        keep = [0, 1, 3]
        for p, q in zip(base, other):
            assert torch.equal(p[keep], q[keep])
        assert not torch.equal(base[0][2], other[0][2])
        # one zero row more: the same step (rec_lr scaled by (m + 1) / m for the normaliser), across the 64-column tile
        a1 = torch.cat([a, torch.zeros(1, 784, device="cuda")])
        y1 = torch.cat([y, torch.zeros(B, 1, device="cuda")], dim=1)
        rec1, loss1, idx1 = gen.reconstruct_measured(y1, a1, R_, L, lr * (m + 1) / m, z_init_val=z0, return_aux=True)
        t = TOL[precision]
        assert float((rec1 - base[0]).abs().max()) <= t["fwd"]
        assert float((loss1 * (m + 1) / m - base[1]).abs().max()) <= t["loss"]
        assert torch.equal(idx1, base[2])
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_steady_state_and_alternating_calls(precision):
    """A second measured call at a planned size allocates nothing and replays its captured loop, with the documented
    launch and enqueue counts; measured, plain and weighted calls alternating on one workspace give the bits of fresh
    handles' calls."""
    arch, B, R_, L, m = "mnist", 5, 3, 7, 100
    w, gen = _gen(arch, precision)
    fresh = []
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(3)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, 784, seed=1)).cuda()
        y = _measure(a, x)

        def call(g, kind):
            if kind == "measured":
                out = g.reconstruct_measured(y, a, R_, L, 1.0, z_init_val=z0, return_aux=True)
            else:
                out = g.reconstruct(x, R_, L, 1.0, z_init_val=z0, return_aux=True,
                                    pixel_weights=pw if kind == "weighted" else None)
            return [t.clone() for t in out]

        want = {}
        for kind in ("measured", "plain", "weighted"):
            _, g = _gen(arch, precision)
            fresh.append(g)
            want[kind] = call(g, kind)
        for kind in ("measured", "plain", "measured", "weighted", "measured", "plain"):
            got = call(gen, kind)
            assert all(torch.equal(p, q) for p, q in zip(got, want[kind])), kind
        call(gen, "plain")
        plain_enq, plain_launches = gen.last_enqueue_count, gen.last_launch_count
        call(gen, "measured")
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        per_step = 6 if precision == "fp16" else 3
        for _ in range(3):
            call(gen, "measured")
            assert gen.last_enqueue_count == plain_enq + 2
            assert gen.last_launch_count == plain_launches + 3 + per_step * (L - 1) + 1
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
        assert plain_enq + 2 <= 12           # the loop is one graph launch, not L-step launches
    finally:
        gen.close()
        for g in fresh:
            g.close()


def test_defensegan_reconstruct_measured_is_the_native_call():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    gan.rec_rr, gan.rec_iters = 2, 5
    x = torch.tensor(O.synthetic_images("mnist", O.init_generator_weights("mnist"), 3)).cuda()
    z0 = torch.randn(6, 128, device="cuda") * 128 ** -0.5
    a = MO.block_average_operator(28, 28, 1, 2)
    y = _measure(torch.tensor(a).cuda(), x)
    got = gan.reconstruct_measured(y.cpu().numpy(), a, z_init_val=z0)
    want = gan._get_native(x.device).reconstruct_measured(y, torch.tensor(a).cuda(), 2, 5, float(gan.rec_lr), z_init_val=z0,
                                                          momentum=float(gan.rec_momentum))
    assert torch.equal(got, want)
    with pytest.raises(ValueError, match="measurements"):
        gan.reconstruct_measured(y[:, :-1], a)
    gan._drop_native()
