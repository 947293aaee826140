"""GPU tests (H100, -m gpu) of generators at widths other than the default latent_dim 128 / net_dim 64, through
DefenseGANBase with the widths as cfg overrides, against the fp64 oracle.  The handle pads every channel width with exact
zeros (fp32 path: to a multiple of 64; fp16 path: to 64, 128, 256 or 512, the Linear's output to at least 256) and splits
fp16 layer-directions wider than 256 channels into column blocks, so the tolerances are those test_gpu_parity.py states for
each precision: the padded sums are the unpadded ones with zero terms appended.

The BatchNorm row's loop is compared at the hyper-parameters and tolerances of test_gpu_parity.py's BatchNorm test
(lr 0.5, L = 3): batch statistics couple the rows, so a restart of nearly the same loss may win on fp16.
CelebA net_dim = 128 on fp32 needs 105,984 B of shared memory in the last layer's forward, more than the 100 KB the
kernel used to opt in to; the largest widths the fp32 path accepts (net_dim 704 on MNIST, 256 on CelebA) run too."""
import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

# (arch, latent_dim, net_dim, use_bn)
ROWS = [("mnist", 100, 32, False), ("mnist", 128, 128, False), ("celeba", 200, 48, False), ("celeba", 64, 128, True)]
TOL = {"fp32": dict(fwd=2e-5, grad_rel=2e-4, grad_cos=0.999999, rec=1e-4, loss=1e-6),
       "fp16": dict(fwd=5e-3, grad_rel=6e-2, grad_cos=0.998, rec=2e-2, loss=1e-4)}


def _model(arch, latent, net_dim, use_bn, precision):
    from defensegan_b200.models.gan import CelebADefenseGAN, MnistDefenseGAN
    cls = CelebADefenseGAN if arch == "celeba" else MnistDefenseGAN
    gan = cls(test_mode=True, verbose=False, precision=precision, latent_dim=latent, net_dim=net_dim, use_bn=use_bn)
    # non-zero biases and BN affine parameters, so that their padding is exercised too
    gan.weights = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, use_bn=use_bn, random_bias=True)
    return gan


@pytest.fixture(scope="module")
def oracle_runs():
    cache = {}

    def get(key, fn):
        if key not in cache:
            cache[key] = fn()
        return cache[key]

    return get


LOOP_ROWS = [r for r in ROWS if not r[3]]
BN_TOL = {"fp32": dict(fwd=5e-5, loss=1e-5, grad_rel=1e-3, rec=1e-3, lmin=1e-4),
          "fp16": dict(fwd=1e-2, loss=1e-3, grad_rel=6e-2, rec=1e-1, lmin=1e-3)}


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", ROWS)
def test_loss_and_grad_match_oracle(arch, latent, net_dim, use_bn, precision):
    """One loop body at B=4, R=2: y = G(z), per-row loss and dL/dz, with the tolerances test_gpu_parity.py states (with
    BatchNorm: those of its BatchNorm test)."""
    gan = _model(arch, latent, net_dim, use_bn, precision)
    try:
        native = gan._get_native(torch.device("cuda", 0))
        B, R = 4, 2
        imgs = O.synthetic_images(arch, gan.weights, B, kind="S2", seed=5, latent_dim=latent)
        z = O.sample_z0(B * R, latent, seed=6)
        y64, loss64, grad64 = O.loss_and_grad(arch, gan.weights, imgs, z, R, use_bn=use_bn, dtype=torch.float64)
        y, loss, grad = native.loss_grad(torch.tensor(imgs).cuda(), torch.tensor(z).cuda(), R)
        t = BN_TOL[precision] if use_bn else TOL[precision]
        # test_gpu_parity.py's loss bound: the forward tolerance carried through the squared error
        ltol = t["loss"] if use_bn else max(t["loss"], 1e-3 * t["fwd"] / 2e-5 * 1e-3)
        yerr = float(np.abs(y.cpu().numpy() - y64).max())
        lerr = float(np.abs(loss.cpu().numpy() - loss64).max())
        g = grad.cpu().numpy()
        gerr = float(np.abs(g - grad64).max() / np.abs(grad64).max())
        print("%s %s latent=%d net_dim=%d bn=%d body: |dy| %.3g |dloss| %.3g grad rel %.3g"
              % (precision, arch, latent, net_dim, use_bn, yerr, lerr, gerr))
        assert g.shape == (B * R, latent)
        assert yerr <= t["fwd"] and lerr <= ltol and gerr <= t["grad_rel"], (yerr, lerr, gerr)
    finally:
        gan.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", LOOP_ROWS)
def test_reconstruct_short_horizon_elementwise(oracle_runs, arch, latent, net_dim, use_bn, precision):
    gan = _model(arch, latent, net_dim, use_bn, precision)
    B, R, L = 16, 2, 10
    gan.rec_rr, gan.rec_iters = R, L
    imgs = O.synthetic_images(arch, gan.weights, B, latent_dim=latent)
    z0 = O.sample_z0(B * R, latent, seed=7)
    try:
        ref = oracle_runs(("short", arch, latent, net_dim), lambda: O.reconstruct(
            arch, gan.weights, imgs, R, L, z_init_val=z0, dtype=torch.float64))
        rec, loss, _ = gan.reconstruct(torch.tensor(imgs).cuda(), z_init_val=torch.tensor(z0).cuda(), return_aux=True)
        t = TOL[precision]
        err = float(np.abs(rec.cpu().numpy() - ref["rec"]).max())
        lerr = float(np.abs(loss.cpu().numpy() - ref["loss_min"]).max())
        print("%s %s latent=%d net_dim=%d: max|rec - oracle64| = %.3g, max|loss - oracle64| = %.3g"
              % (precision, arch, latent, net_dim, err, lerr))
        assert err <= t["rec"] and lerr <= t["loss"], (err, lerr)
    finally:
        gan.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_batchnorm_row_reconstruct(precision):
    """CelebA latent 64 / net_dim 128 with BatchNorm: the loop at test_gpu_parity.py's BatchNorm hyper-parameters, with its
    tolerances: every restart the oracle's on fp32 (at least half on fp16), the images of agreeing restarts and the
    per-image loss within the stated bounds."""
    arch, latent, net_dim = "celeba", 64, 128
    gan = _model(arch, latent, net_dim, True, precision)
    B, R, L, lr = 8, 2, 3, 0.5
    gan.rec_rr, gan.rec_iters, gan.rec_lr = R, L, lr
    imgs = O.synthetic_images(arch, gan.weights, B, latent_dim=latent)
    z0 = O.sample_z0(B * R, latent, seed=7)
    try:
        ref = O.reconstruct(arch, gan.weights, imgs, R, L, rec_lr=lr, z_init_val=z0, use_bn=True, dtype=torch.float64)
        rec, lmin, idx = gan.reconstruct(torch.tensor(imgs).cuda(), z_init_val=torch.tensor(z0).cuda(), return_aux=True)
        t = BN_TOL[precision]
        agree = idx.cpu().numpy() == ref["idx"]
        drec = np.abs(rec.cpu().numpy() - ref["rec"]).reshape(B, -1).max(axis=1)
        rerr = float(drec[agree].max()) if agree.any() else 0.0
        merr = float(np.abs(lmin.cpu().numpy() - ref["loss_min"]).max())
        print("%s BN row: |drec| %.3g (restart agreement %.2f) |dloss_min| %.3g" % (precision, rerr, agree.mean(), merr))
        assert agree.all() if precision == "fp32" else agree.mean() >= 0.5
        assert rerr <= t["rec"] and merr <= t["lmin"], (rerr, merr)
    finally:
        gan.close()


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", LOOP_ROWS)
def test_long_horizon_per_image_mse(arch, latent, net_dim, use_bn):
    """L = 200 (the metric's operating point): per-image |MSE_min - oracle64| <= 1e-4 on every precision that serves the
    width."""
    B, R, L = 4, 4, 200
    w = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, use_bn=use_bn, random_bias=True)
    imgs = O.synthetic_images(arch, w, B, latent_dim=latent)
    z0 = O.sample_z0(B * R, latent, seed=8)
    ref = O.reconstruct(arch, w, imgs, R, L, z_init_val=z0, use_bn=use_bn, dtype=torch.float64)
    for precision in ("fp32", "fp16"):
        gan = _model(arch, latent, net_dim, use_bn, precision)
        gan.rec_rr, gan.rec_iters = R, L
        try:
            _, loss, _ = gan.reconstruct(torch.tensor(imgs).cuda(), z_init_val=torch.tensor(z0).cuda(), return_aux=True)
            d = float(np.abs(loss.cpu().numpy() - ref["loss_min"]).max())
            print("%s %s latent=%d net_dim=%d bn=%d L=200: max|dMSE| = %.3g" % (precision, arch, latent, net_dim, use_bn, d))
            assert d <= 1e-4, d
        finally:
            gan.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [ROWS[0], ROWS[1], ROWS[2]])
def test_generator_fn_forward_and_vjp(arch, latent, net_dim, use_bn, precision):
    """generator_fn(z) and its torch.autograd backward (dgan_vjp): dz comes back at the real latent width."""
    gan = _model(arch, latent, net_dim, use_bn, precision)
    try:
        n = 6
        z = torch.tensor(O.sample_z0(n, latent, seed=9)).cuda().requires_grad_(True)
        y = gan.generator_fn(z)
        dy = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda()
        y.backward(dy)
        w64 = O.weights_to_torch(gan.weights, torch.float64)
        z64 = z.detach().cpu().double().requires_grad_(True)
        y64 = O.generator_forward(arch, w64, z64, use_bn=use_bn)
        (g64,) = torch.autograd.grad(y64, z64, dy.cpu().double())
        t = TOL[precision]
        assert z.grad.shape == (n, latent)
        assert float((y.detach().cpu().double() - y64.detach()).abs().max()) <= t["fwd"]
        g, g64 = z.grad.cpu().double().numpy(), g64.numpy()
        gerr = np.abs(g - g64).max() / np.abs(g64).max()
        cos = float((g * g64).sum() / np.sqrt((g * g).sum() * (g64 * g64).sum()))
        assert gerr <= t["grad_rel"] and cos >= t["grad_cos"], (gerr, cos)
    finally:
        gan.close()


def _philox_z0(seed, first_elem, n, latent):
    """The z0 draw by its definition: element e of the row-major [rows, latent] array is value e % 4 of Philox4x32-10
    block e / 4 (counter (e / 4) as 64 bits, key = seed), through Box-Muller, times sqrt(1 / latent)."""
    M = np.uint64(0xFFFFFFFF)
    e = np.arange(first_elem, first_elem + n, dtype=np.uint64)
    q = e // np.uint64(4)
    c0, c1 = q & M, q >> np.uint64(32)
    c2 = np.zeros_like(c0)
    c3 = np.zeros_like(c0)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    u = [(r.astype(np.float32) + np.float32(0.5)) * np.float32(2.3283064365386963e-10) for r in (c0, c1, c2, c3)]
    lane = (e % np.uint64(4)).astype(np.int64)
    ua = np.where(lane < 2, u[0], u[2]).astype(np.float64)
    ub = np.where(lane < 2, u[1], u[3]).astype(np.float64)
    m = np.sqrt(-2.0 * np.log(ua)) * np.sqrt(1.0 / latent)
    return np.where(lane % 2 == 1, m * np.sin(2 * np.pi * ub), m * np.cos(2 * np.pi * ub))


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_z0_is_drawn_by_real_index(precision):
    """At latent 100 (padded to 128) dgan_sample_z0 is the Philox draw indexed by the real (row, column), and the draw
    inside dgan_reconstruct is the same one: the padding does not show."""
    latent, seed, off = 100, 1234567, 5
    gan = _model("mnist", latent, 32, False, precision)
    try:
        native = gan._get_native(torch.device("cuda", 0))
        z = native.sample_z0(37, seed, z_row_offset=off).cpu().numpy()
        want = _philox_z0(seed, off * latent, 37 * latent, latent).reshape(37, latent)
        assert float(np.abs(z - want).max()) <= 1e-6
        B, R = 3, 4
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, B, latent_dim=latent)).cuda()
        a = native.reconstruct(x, R, 5, 10.0, seed=seed, z_row_offset=off)
        b = native.reconstruct(x, R, 5, 10.0, z_init_val=native.sample_z0(B * R, seed, z_row_offset=off))
        assert torch.equal(a, b)
    finally:
        gan.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_steady_state_calls_do_not_allocate(precision):
    gan = _model("celeba", 200, 48, False, precision)
    try:
        native = gan._get_native(torch.device("cuda", 0))
        B, R = 3, 2
        x = torch.tensor(O.synthetic_images("celeba", gan.weights, B, latent_dim=200)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R, 200)).cuda()
        want = native.reconstruct(x, R, 7, 1.0, z_init_val=z0).clone()
        assert torch.equal(native.reconstruct(x, R, 7, 1.0, z_init_val=z0), want)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for _ in range(3):
            assert torch.equal(native.reconstruct(x, R, 7, 1.0, z_init_val=z0), want)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
    finally:
        gan.close()


def _exact_macs(arch, latent, nd):
    """SURVEY Appendix B: in-bounds tap pairs per axis of a 5x5 / stride-2 transposed conv on an H-pixel input are 5H - 3
    (15 for MNIST's 4 -> 7 crop); MACs = pairs^2 * C_in * C_out, at the real widths."""
    if arch == "mnist":
        return latent * 16 * 4 * nd + 15 ** 2 * 4 * nd * 2 * nd + 32 ** 2 * 2 * nd * nd + 67 ** 2 * nd
    return latent * 16 * 4 * nd + 17 ** 2 * 8 * nd * nd + 37 ** 2 * 2 * nd * nd + 77 ** 2 * nd * nd + 157 ** 2 * nd * 3


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [r for r in ROWS if not r[3]])
def test_macs_per_row_count_the_real_widths(arch, latent, net_dim, use_bn):
    for precision in ("fp32", "fp16"):
        gan = _model(arch, latent, net_dim, use_bn, precision)
        try:
            assert gan._get_native(torch.device("cuda", 0)).macs_per_row == _exact_macs(arch, latent, net_dim)
        finally:
            gan.close()


@pytest.mark.parametrize("arch,net_dim", [("mnist", 704), ("celeba", 256)])
def test_fp32_runs_at_its_largest_accepted_width(arch, net_dim):
    """The last layer's forward then needs 228,992 B (MNIST) or 209,920 B (CelebA) of the shared memory it opts in to: G(z)
    matches the oracle and a short reconstruct runs."""
    latent = 100
    gan = _model(arch, latent, net_dim, False, "fp32")
    try:
        z = torch.tensor(O.sample_z0(2, latent, seed=9)).cuda()
        y = gan.generator_fn(z)
        w64 = O.weights_to_torch(gan.weights, torch.float64)
        y64 = O.generator_forward(arch, w64, z.cpu().double())
        err = float((y.cpu().double() - y64).abs().max())
        print("fp32 %s net_dim=%d: max|G(z) - oracle64| = %.3g" % (arch, net_dim, err))
        assert err <= TOL["fp32"]["fwd"], err
        gan.rec_rr, gan.rec_iters = 1, 2
        rec, loss, _ = gan.reconstruct(y.detach(), z_init_val=z, return_aux=True)
        assert rec.shape == y.shape and bool(torch.isfinite(loss).all())
    finally:
        gan.close()
