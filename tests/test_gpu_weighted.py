"""GPU tests (H100, -m gpu) of the per-pixel weighted projection (dgan_reconstruct_weighted, dgan_loss_grad_weighted):
  - weights of 1 give the unweighted call's bits (rec, loss, idx; y, loss, grad) on both precisions, MNIST and CelebA,
    with and without BatchNorm;
  - the images' pixels of weight 0 do not change a bit of any output;
  - random weights in [0, 1] and binary masks at R = 10, L = 200 against the weighted CPU oracle (tests/weighted_oracle.py)
    within test_gpu_parity.py's tolerances, and one loss / gradient evaluation against its fp64 evaluation;
  - each layer-direction of a weighted dgan_loss_grad against fp64 on the operands the kernels read (tests/layer_ref.py,
    tests/weighted_layer_ref.py);
  - steady state: no allocation, the captured loop replayed, one stream operation more than the unweighted call, and
    weighted and unweighted calls alternating on one workspace give the bits of fresh calls."""
import numpy as np
import pytest
import torch

import layer_ref as R
import weighted_layer_ref as WR
import weighted_oracle as WO
from gpu_support import gen as _gen, layout, read_call, release_cached_memory, view  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


TOL = {"fp32": dict(fwd=2e-5, grad_rel=2e-4, grad_cos=0.999999, loss=1e-6),
       "fp16": dict(fwd=5e-3, grad_rel=6e-2, grad_cos=0.998, loss=1e-4)}


def _weights(shape, kind, seed=0):
    rs = np.random.RandomState(seed)
    if kind == "ones":
        return np.ones(shape, dtype=np.float32)
    if kind == "mask":
        w = np.ones(shape, dtype=np.float32)
        h = shape[1]
        for i in range(shape[0]):                 # an occluded square per image, at a random place
            r, c = rs.randint(0, h // 2, size=2)
            w[i, r:r + h // 2, c:c + h // 2] = 0
        return w
    w = rs.uniform(0, 1, size=shape).astype(np.float32)
    w[rs.uniform(size=shape) < 0.1] = 0
    return w


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_unit_weights_give_the_unweighted_bits(precision, arch, use_bn):
    w, gen = _gen(arch, precision, use_bn)
    try:
        B, R_, L = 3, 2, 6
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        ones = torch.ones_like(x)
        plain = gen.reconstruct(x, R_, L, 10.0, z_init_val=z0, return_aux=True)
        weighted = gen.reconstruct(x, R_, L, 10.0, z_init_val=z0, return_aux=True, pixel_weights=ones)
        for a, b in zip(plain, weighted):
            assert torch.equal(a, b)
        for a, b in zip(gen.loss_grad(x, z0, R_), gen.loss_grad(x, z0, R_, pixel_weights=ones)):
            assert torch.equal(a, b)
    finally:
        gen.close()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_pixels_of_weight_zero_change_nothing(precision, arch):
    w, gen = _gen(arch, precision)
    try:
        B, R_, L = 4, 3, 8
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        pw = torch.tensor(_weights(tuple(x.shape), "mask", seed=1)).cuda()
        x2 = torch.where(pw == 0, torch.rand_like(x), x)
        assert not torch.equal(x, x2)
        for a, b in zip(gen.reconstruct(x, R_, L, 10.0, z_init_val=z0, return_aux=True, pixel_weights=pw),
                        gen.reconstruct(x2, R_, L, 10.0, z_init_val=z0, return_aux=True, pixel_weights=pw)):
            assert torch.equal(a, b)
        for a, b in zip(gen.loss_grad(x, z0, R_, pixel_weights=pw), gen.loss_grad(x2, z0, R_, pixel_weights=pw)):
            assert torch.equal(a, b)
    finally:
        gen.close()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_weighted_loss_and_grad_match_oracle(precision, arch):
    w, gen = _gen(arch, precision)
    try:
        B, R_ = 3, 2
        imgs = O.synthetic_images(arch, w, B, kind="S2", seed=5)
        z = O.sample_z0(B * R_, 128, seed=6)
        pw = _weights(imgs.shape, "uniform", seed=7)
        y64, loss64, grad64 = WO.loss_and_grad(arch, w, imgs, z, R_, dtype=torch.float64, pixel_weights=pw)
        y, loss, grad = gen.loss_grad(torch.tensor(imgs).cuda(), torch.tensor(z).cuda(), R_, pixel_weights=torch.tensor(pw).cuda())
        t = TOL[precision]
        assert np.abs(y.cpu().numpy() - y64).max() <= t["fwd"]
        assert np.abs(loss.cpu().numpy() - loss64).max() <= max(t["loss"], 1e-3 * t["fwd"] / 2e-5 * 1e-3)
        g = grad.cpu().numpy()
        assert np.abs(g - grad64).max() / np.abs(grad64).max() <= t["grad_rel"]
        assert float((g * grad64).sum() / np.sqrt((g * g).sum() * (grad64 * grad64).sum())) >= t["grad_cos"]
    finally:
        gen.close()


_ORACLE = {}


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("kind", ["uniform", "mask"])
def test_long_horizon_weighted_parity(precision, kind):
    """R = 10, L = 200 (the metric's operating point), MNIST, 8 images: per-image |loss_min - oracle| <= 1e-4, the bar of
    test_gpu_parity.py's long-horizon test, on the weighted loss."""
    arch, B, R_, L = "mnist", 8, 10, 200
    w, gen = _gen(arch, precision)
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R_, 128)
        pw = _weights(imgs.shape, kind, seed=11)
        if kind not in _ORACLE:
            _ORACLE[kind] = WO.reconstruct(arch, w, imgs, R_, L, z_init_val=z0, pixel_weights=pw)
        ref = _ORACLE[kind]
        rec, loss, idx = gen.reconstruct(torch.tensor(imgs).cuda(), R_, L, 10.0, z_init_val=torch.tensor(z0).cuda(),
                                         return_aux=True, pixel_weights=torch.tensor(pw).cuda())
        dmse = np.abs(loss.cpu().numpy() - ref["loss_min"])
        agree = float((idx.cpu().numpy() == ref["idx"]).mean())
        print("precision=%s weights=%s max|dloss|=%.3g restart agreement=%.2f" % (precision, kind, dmse.max(), agree))
        assert dmse.max() <= 1e-4
        # the returned loss is the weighted MSE of the returned reconstruction
        wl = (torch.tensor(pw).cuda() * (rec - torch.tensor(imgs).cuda()) ** 2).mean(dim=(1, 2, 3))
        assert float((wl - loss).abs().max()) <= 1e-6
    finally:
        gen.close()


# (arch, latent_dim, net_dim, use_bn)
LAYER_MATRIX = [("mnist", 128, 64, False), ("mnist", 128, 64, True), ("celeba", 128, 64, False), ("celeba", 64, 128, True)]


@pytest.mark.parametrize("n_rows", [1, 300, 2560])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", LAYER_MATRIX)
def test_weighted_loss_grad_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows):
    w, gen = _gen(arch, precision, use_bn, latent, net_dim)
    try:
        R_ = 1 if n_rows == 1 else 2
        B = n_rows // R_
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3, latent_dim=latent)).cuda()
        pw = torch.tensor(_weights(tuple(imgs.shape), "uniform", seed=8)).cuda()
        z = torch.tensor(O.sample_z0(n_rows, latent, seed=4)).cuda()
        gen.loss_grad(imgs, z, R_, pixel_weights=pw)
        torch.cuda.synchronize()
        x_rows = imgs.reshape(B, -1).repeat_interleave(R_, dim=0)
        w_rows = pw.reshape(B, -1).repeat_interleave(R_, dim=0)
        ws, net = read_call(gen, w, arch, latent, net_dim, use_bn, precision, n_rows)
        stats = R.Stats()
        R.check_inputs(net, ws, n_rows, z)
        R.check_forward(net, ws, n_rows, stats, "")
        WR.check_last_fwd_weighted(net, ws, n_rows, x_rows, w_rows, stats, "")
        R.check_backward(net, ws, n_rows, stats, "")
        print("\nweighted %s %s latent=%d net_dim=%d bn=%d rows=%d" % (precision, arch, latent, net_dim, use_bn, n_rows))
        print("\n".join(stats.lines()))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_steady_state_and_alternating_calls(precision):
    """A second weighted call at a planned size allocates nothing, replays its captured loop and issues one stream
    operation more than the unweighted call (the weight copy); weighted and unweighted calls alternating on one workspace
    give the bits of fresh handles' calls."""
    arch, B, R_, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    fresh = []
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        pw = torch.tensor(_weights(tuple(x.shape), "uniform", seed=3)).cuda()

        def call(g, weighted):
            return [t.clone() for t in g.reconstruct(x, R_, L, 1.0, z_init_val=z0, return_aux=True,
                                                     pixel_weights=pw if weighted else None)]

        want = {}
        for weighted in (True, False):
            _, g = _gen(arch, precision)
            fresh.append(g)
            want[weighted] = call(g, weighted)
        for weighted in (True, False, True, False, True):
            got = call(gen, weighted)
            assert all(torch.equal(a, b) for a, b in zip(got, want[weighted])), weighted
        assert not torch.equal(want[True][0], want[False][0])
        call(gen, False)
        plain = gen.last_enqueue_count
        call(gen, True)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        launches = gen.last_launch_count
        for _ in range(3):
            call(gen, True)
            assert gen.last_enqueue_count == plain + 1 and gen.last_launch_count == launches
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
        assert plain + 1 <= 11         # the loop is one graph launch, not L-step launches
        # the weighted layout: the unweighted buffers at their offsets, then the copy of the weights the loop read
        plain_ws = layout(gen, "", B * R_)[1].splitlines()
        regions, weighted_ws = layout(gen, "_weighted", B * R_)
        weighted_ws = weighted_ws.splitlines()
        assert weighted_ws[:len(plain_ws)] == plain_ws and weighted_ws[len(plain_ws)].split()[0] == "xw"
        xw = view(gen, regions[0], weighted_ws[-1].split()[0])
        assert torch.equal(xw[:B], pw.reshape(B, -1))
    finally:
        gen.close()
        for g in fresh:
            g.close()


def test_defensegan_reconstruct_with_a_broadcast_mask():
    """DefenseGANBase.reconstruct: an [H, W, C] mask broadcasts to every image; the result is the native weighted call's."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    gan.rec_rr, gan.rec_iters = 2, 5
    x = torch.tensor(O.synthetic_images("mnist", O.init_generator_weights("mnist"), 3)).cuda()
    z0 = torch.randn(6, 128, device="cuda") * 128 ** -0.5
    mask = np.ones((28, 28, 1), dtype=np.float32)
    mask[10:20, 5:15] = 0
    got = gan.reconstruct(x, z_init_val=z0, pixel_weights=mask)
    native = gan._get_native(x.device)
    want = native.reconstruct(x, 2, 5, float(gan.rec_lr), z_init_val=z0, momentum=float(gan.rec_momentum),
                              pixel_weights=torch.tensor(mask).cuda().expand_as(x).contiguous())
    assert torch.equal(got, want)
    with pytest.raises(ValueError):
        gan.reconstruct(x, z_init_val=z0, pixel_weights=mask * 2)
    gan._drop_native()
