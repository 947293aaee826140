"""GPU parity tests (run on an H100 with -m gpu): every call goes through the C-ABI
(ctypes -> libdefensegan_b200.so) and is checked against the CPU oracle / golden vectors.

Tolerances (stated per precision):
  fp32 (CUDA-core FMA, the reference's arithmetic type): elementwise |rec - rec_oracle64| <= 1e-4,
       identical arg-min indices, |loss_min - oracle| <= 1e-6 at the C1 horizon.
  fp16 (wgmma operands, fp32 accumulate): per-image |MSE_min - oracle| <= 1e-4 (BASELINE.json's
       bar), elementwise |rec - rec_oracle| <= 2e-2 at the C1 horizon.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from gpu_support import ws_base
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "fp16"]
TOL = {
    "fp32": dict(fwd=2e-5, grad_rel=2e-4, grad_cos=0.999999, rec=1e-4, loss=1e-6),
    # fp16 gradient: rounding flips the ReLU mask of units whose pre-activation is ~0, which moves the
    # gradient by finite (not rounding-sized) amounts: a few % of max |g| while the direction stays put
    "fp16": dict(fwd=5e-3, grad_rel=6e-2, grad_cos=0.998, rec=2e-2, loss=1e-4),
}


def _native_gen(arch, weights, precision):
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    tensors = [torch.as_tensor(v).to(dev) for v in weights.values()]
    return _native.NativeGenerator(arch, tensors, precision=precision, device=dev)


@pytest.fixture(scope="module")
def gens():
    cache = {}

    def get(arch, precision, random_bias=False):
        key = (arch, precision, random_bias)
        if key not in cache:
            w = O.init_generator_weights(arch, random_bias=random_bias)
            cache[key] = (w, _native_gen(arch, w, precision))
        return cache[key]

    yield get
    for _, g in cache.values():
        g.close()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_forward_matches_oracle(gens, arch, precision):
    w, gen = gens(arch, precision, True)
    z = O.sample_z0(5, 128, seed=3)
    want = O.generator_forward(arch, O.weights_to_torch(w, torch.float64), torch.tensor(z, dtype=torch.float64)).numpy()
    got = gen.forward(torch.tensor(z).cuda()).cpu().numpy()
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= TOL[precision]["fwd"]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_loss_and_grad_match_oracle(gens, arch, precision):
    w, gen = gens(arch, precision, True)
    B, R = 3, 2
    imgs = O.synthetic_images(arch, w, B, kind="S2", seed=5)
    z = O.sample_z0(B * R, 128, seed=6)
    y64, loss64, grad64 = O.loss_and_grad(arch, w, imgs, z, R, dtype=torch.float64)
    y, loss, grad = gen.loss_grad(torch.tensor(imgs).cuda(), torch.tensor(z).cuda(), R)
    t = TOL[precision]
    assert np.abs(y.cpu().numpy() - y64).max() <= t["fwd"]
    assert np.abs(loss.cpu().numpy() - loss64).max() <= max(t["loss"], 1e-3 * t["fwd"] / 2e-5 * 1e-3)
    g = grad.cpu().numpy()
    gerr = np.abs(g - grad64).max() / np.abs(grad64).max()
    cos = float((g * grad64).sum() / np.sqrt((g * g).sum() * (grad64 * grad64).sum()))
    assert gerr <= t["grad_rel"], gerr
    assert cos >= t["grad_cos"], cos


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", ["mnist_c1", "mnist_ragged_bias", "celeba_small"])
def test_reconstruct_matches_golden(gens, golden_dir, case, precision):
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    arch = str(g["arch"])
    w, gen = gens(arch, precision, bool(int(g["random_bias"])))
    rec, loss, idx = gen.reconstruct(torch.tensor(g["images"]).cuda(), int(g["R"]), int(g["L"]), float(g["lr"]),
                                     z_init_val=torch.tensor(g["z0"]).cuda(), return_aux=True)
    rec, loss, idx = rec.cpu().numpy(), loss.cpu().numpy(), idx.cpu().numpy()
    t = TOL[precision]
    assert rec.shape == g["images"].shape
    np.testing.assert_array_equal(idx, g["idx64"])
    assert np.abs(loss - g["loss_min64"]).max() <= t["loss"]
    assert np.abs(rec - g["rec64"]).max() <= t["rec"]
    # and against the fp32 oracle run (the reference-precision stand-in)
    assert np.abs(rec - g["rec32"]).max() <= t["rec"]


@pytest.mark.parametrize("precision", PRECISIONS)
def test_size_independent_properties_at_full_size(gens, precision):
    """BASELINE configs[1] size (B=256, R=10) at a shortened horizon plus properties that need no
    oracle: run-to-run bit-exactness, loss_min == MSE(rec, x), tie -> lowest index, batch-split
    invariance (== what sharding across GPUs relies on)."""
    arch = "mnist"
    w, gen = gens(arch, precision)
    B, R, L = 256, 10, 12
    x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
    z0 = torch.tensor(O.sample_z0(B * R, 128)).cuda()
    rec, loss, idx = gen.reconstruct(x, R, L, 10.0, z_init_val=z0, return_aux=True)
    rec2, loss2, idx2 = gen.reconstruct(x, R, L, 10.0, z_init_val=z0, return_aux=True)
    assert torch.equal(rec, rec2) and torch.equal(loss, loss2) and torch.equal(idx, idx2)
    mse = ((rec - x) ** 2).mean(dim=(1, 2, 3))
    assert float((mse - loss).abs().max()) <= 1e-6
    assert int(idx.min()) >= 0 and int(idx.max()) < R and len(torch.unique(idx)) > 1
    # the projection must actually descend: loss after L steps < loss of the best initial restart
    _, loss_l1, _ = gen.reconstruct(x, R, 1, 10.0, z_init_val=z0, return_aux=True)
    assert float(loss.mean()) < float(loss_l1.mean())
    # batch-split invariance (rows are independent without BatchNorm)
    h = 96
    rec_a = gen.reconstruct(x[:h], R, L, 10.0, z_init_val=z0[:h * R])
    rec_b = gen.reconstruct(x[h:], R, L, 10.0, z_init_val=z0[h * R:])
    assert torch.equal(torch.cat([rec_a, rec_b]), rec)
    # identical restarts tie -> index 0 (tf.argmin)
    z_tie = z0.view(B, R, -1)[:, :1].expand(B, R, 128).reshape(B * R, 128).contiguous()
    _, _, idx_tie = gen.reconstruct(x, R, 3, 10.0, z_init_val=z_tie, return_aux=True)
    assert int(idx_tie.abs().max()) == 0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_long_horizon_statistical_parity(gens, precision):
    """L=200, R=10 (the metric's operating point) on a batch the oracle finishes in ~20 s:
    per-image |MSE_min - oracle_fp32| <= 1e-4 (BASELINE.json), restart agreement reported."""
    arch = "mnist"
    w, gen = gens(arch, precision)
    B, R, L = 8, 10, 200
    imgs = O.synthetic_images(arch, w, B)
    z0 = O.sample_z0(B * R, 128)
    ref = O.reconstruct(arch, w, imgs, R, L, z_init_val=z0)
    rec, loss, idx = gen.reconstruct(torch.tensor(imgs).cuda(), R, L, 10.0, z_init_val=torch.tensor(z0).cuda(),
                                     return_aux=True)
    dmse = np.abs(loss.cpu().numpy() - ref["loss_min"])
    agree = float((idx.cpu().numpy() == ref["idx"]).mean())
    print("precision=%s max|dMSE|=%.3g restart agreement=%.2f" % (precision, dmse.max(), agree))
    assert dmse.max() <= 1e-4


@pytest.mark.parametrize("precision", PRECISIONS)
def test_python_surface_and_random_restarts(precision):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils.gan_defense import model_eval_gan, SharedReconstruction
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision=precision)
    assert gan.load_generator() is False          # no checkpoint: keeps reference-style random init
    gan.rec_rr, gan.rec_iters = 4, 5
    x = torch.tensor(O.synthetic_images("mnist", gan.weights, 6)).cuda()
    a = gan.reconstruct(x)
    b = gan.reconstruct(x)
    assert a.shape == x.shape and a.is_cuda and not a.requires_grad
    assert not torch.equal(a, b)                  # fresh z0 per call (utils/gan_defense.py:119)
    z0 = torch.tensor(O.sample_z0(6 * 4, 128)).cuda()
    assert torch.equal(gan.reconstruct(x, z_init_val=z0), gan.reconstruct(x, z_init_val=z0))
    with pytest.raises(ValueError):
        gan.reconstruct(x[:, :14])
    labels = np.eye(10, dtype="f4")[np.arange(6) % 10]
    rec = SharedReconstruction(gan)
    clf = torch.nn.Linear(784, 10).cuda()
    acc, roc = model_eval_gan(None, None, None, predictions=lambda xb: clf(rec(xb).reshape(len(xb), -1)),
                              test_images=x.cpu().numpy(), test_labels=labels, args={"batch_size": 4},
                              diff_op=lambda xb: ((xb - rec(xb)) ** 2).mean(dim=(1, 2, 3)))
    assert 0.0 <= acc <= 1.0 and roc[2].shape == (6,) and np.all(roc[2] > 0)
    gan.close()


def test_error_paths_through_c_abi(gens):
    from defensegan_b200 import _native
    w, gen = gens("mnist", "fp32")
    lib = gen.lib
    x = torch.zeros(2, 28, 28, 1, device="cuda")
    rec = torch.empty_like(x)
    small = torch.empty(4096, dtype=torch.uint8, device="cuda")
    base = ws_base(small)
    prm = _native.dgan_rec_params(2, 2, 3, 10.0, 0.7, 0, 0, 0)
    rc = lib.dgan_reconstruct(gen._handle, ctypes.byref(prm), x.data_ptr(), None, rec.data_ptr(), None, None,
                              ctypes.c_void_p(base), 1024, None)
    assert rc == -4 and b"workspace" in lib.dgan_last_error()
    prm.batch = 0
    rc = lib.dgan_reconstruct(gen._handle, ctypes.byref(prm), x.data_ptr(), None, rec.data_ptr(), None, None,
                              ctypes.c_void_p(base), 1024, None)
    assert rc == -1
    assert lib.dgan_reconstruct(gen._handle, None, x.data_ptr(), None, rec.data_ptr(), None, None,
                                ctypes.c_void_p(base), 1024, None) == -1


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("case", ["mnist_bn", "celeba_bn"])
def test_batchnorm_batch_statistics_path(golden_dir, case, precision):
    """use_bn=True (opt-in; tflib/ops/batchnorm.py:80-93 else-branch): batch statistics couple all rows
    (SURVEY F2).  Both paths vs the fp64 oracle: forward/loss/grad of one loop body and the short loop.  On the tensor-core
    path the GEMMs write fp16 pre-activations, the statistics and the normalisation are fp32 arithmetic on them."""
    from defensegan_b200 import _native
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    arch, B, R, L = str(g["arch"]), int(g["B"]), int(g["R"]), int(g["L"])
    w = O.init_generator_weights(arch, random_bias=True, use_bn=True)
    dev = torch.device("cuda", 0)
    gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], use_bn=True, precision=precision,
                                  device=dev)
    t = {"fp32": dict(y=5e-5, loss=1e-5, grad=1e-3, rec=1e-3, lmin=1e-4),
         # fp16 operands: the batch statistics couple the rounding of every row into every row and L steps of lr 10 carry
         # it along - the loss of the chosen restart stays within ~1e-4, single pixels of a CelebA image move by a few 1e-2
         "fp16": dict(y=1e-2, loss=1e-3, grad=6e-2, rec=1e-1, lmin=1e-3)}[precision]
    x, z0 = torch.tensor(g["images"]).cuda(), torch.tensor(g["z0"]).cuda()
    y, loss, grad = gen.loss_grad(x, z0, R)
    yerr, lerr = np.abs(y.cpu().numpy() - g["y0_64"]).max(), np.abs(loss.cpu().numpy() - g["loss0_64"]).max()
    gerr = np.abs(grad.cpu().numpy() - g["grad0_64"]).max() / np.abs(g["grad0_64"]).max()
    rec, lmin, idx = gen.reconstruct(x, R, L, float(g["lr"]), z_init_val=z0, return_aux=True)
    agree = idx.cpu().numpy() == g["idx64"]          # fp16 may pick another restart of (nearly) the same loss: compare
    drec = np.abs(rec.cpu().numpy() - g["rec64"]).reshape(B, -1).max(axis=1)   # images where the restart is the oracle's
    rerr, merr = float(drec[agree].max()) if agree.any() else 0.0, np.abs(lmin.cpu().numpy() - g["loss_min64"]).max()
    print("%s %s BN: |dy| %.2e |dloss| %.2e grad rel %.2e |drec| %.2e (restart agreement %.2f) |dloss_min| %.2e"
          % (case, precision, yerr, lerr, gerr, rerr, agree.mean(), merr))
    assert yerr <= t["y"] and lerr <= t["loss"] and gerr <= t["grad"], (yerr, lerr, gerr)
    assert agree.all() if precision == "fp32" else agree.mean() >= 0.5
    assert rerr <= t["rec"] and merr <= t["lmin"], (rerr, merr)
    # rows are coupled: dropping one image changes the others' reconstructions (unlike the no-BN path)
    rec_sub = gen.reconstruct(x[:-1], R, L, float(g["lr"]), z_init_val=z0[:-R])
    assert not torch.equal(rec_sub, rec[:-1])
    gen.close()


def test_shape_fuzz_ragged_sizes(gens):
    """Any B / R / L (superset of the reference's static shapes, SURVEY F10): tile padding, ragged CTA-pair
    tiles and window schedules for many row counts, fp16 and fp32, against the fp32 oracle."""
    rs = np.random.RandomState(7)
    for trial in range(6):
        B, R, L = int(rs.randint(1, 40)), int(rs.randint(1, 6)), int(rs.randint(1, 4))
        arch = "mnist" if trial % 3 else "celeba"
        if arch == "celeba":
            B = min(B, 6)
        for precision in PRECISIONS:
            w, gen = gens(arch, precision, True)
            imgs = O.synthetic_images(arch, w, B, kind="S2", seed=100 + trial)
            z0 = O.sample_z0(B * R, 128, seed=200 + trial)
            ref = O.reconstruct(arch, w, imgs, R, L, rec_lr=1.0, z_init_val=z0)
            rec, loss, idx = gen.reconstruct(torch.tensor(imgs).cuda(), R, L, 1.0, z_init_val=torch.tensor(z0).cuda(),
                                             return_aux=True)
            t = TOL[precision]
            assert rec.shape == imgs.shape
            assert np.abs(rec.cpu().numpy() - ref["rec"]).max() <= t["rec"], (arch, B, R, L, precision)
            assert np.abs(loss.cpu().numpy() - ref["loss_min"]).max() <= max(t["loss"], 1e-5)


def test_launch_count_and_no_allocation_in_steady_state(gens):
    """What dgan_reconstruct enqueues: z0 initialiser + 4 forward kernels per L-step + 4 backward kernels (the last of them
    applies the momentum update in its tail) per L-step but the last (SURVEY F4) + loss sum + arg-min select; and once a
    batch size has been planned (dgan_workspace_bytes, first call) a call neither allocates nor frees device memory."""
    for arch, per_step in (("mnist", 8), ("celeba", 10)):
        w, gen = gens(arch, "fp16")
        B, R = 3, 2
        x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R, 128)).cuda()
        for L in (1, 2, 7):
            gen.reconstruct(x, R, L, 1.0, z_init_val=z0)
            assert gen.last_launch_count == 1 + per_step // 2 + (L - 1) * per_step + 2, (arch, L, gen.last_launch_count)
        want = gen.reconstruct(x, R, 7, 1.0, z_init_val=z0).clone()
        assert torch.equal(gen.reconstruct(x, R, 7, 1.0, z_init_val=z0), want)      # (also warms torch's own allocator)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for _ in range(3):
            got = gen.reconstruct(x, R, 7, 1.0, z_init_val=z0)
            # the L-step loop is replayed as one CUDA graph: z0 init (+ memsets), image copy, graph, loss sum, select
            assert gen.last_enqueue_count <= 10 and gen.last_launch_count == 1 + per_step // 2 + 6 * per_step + 2
            assert torch.equal(got, want)
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0


def test_graph_cache_survives_many_configurations(gens):
    """The captured L-step loops are cached per (workspace, batch, R, L, lr, momentum, decay) with a small bound: cycling
    through more configurations than the cache holds keeps giving the results of a cold handle's first call."""
    w, gen = gens("mnist", "fp16")
    x = torch.tensor(O.synthetic_images("mnist", w, 4)).cuda()
    z0 = torch.tensor(O.sample_z0(4 * 2, 128)).cuda()
    first = {}
    for sweep in range(2):
        for L in range(1, 12):                                   # 11 loop lengths > 8 cached graphs
            for lr in (1.0, 2.0) if L == 3 else (1.0,):
                rec = gen.reconstruct(x, 2, L, lr, z_init_val=z0).clone()
                if sweep == 0:
                    first[(L, lr)] = rec
                else:
                    assert torch.equal(rec, first[(L, lr)]), (L, lr)
    ref = O.reconstruct("mnist", w, x.cpu().numpy(), 2, 11, rec_lr=1.0, z_init_val=z0.cpu().numpy())
    assert np.abs(first[(11, 1.0)].cpu().numpy() - ref["rec"]).max() <= TOL["fp16"]["rec"]


def test_sharded_api_single_rank_and_random_z0_statistics():
    """parallel.reconstruct_sharded degenerates to the single-GPU call without a process group; the Philox z0
    (models/gan.py:370-377: N(0, 1/latent_dim)) does not depend on how rows are tiled."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.parallel import reconstruct_sharded
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    gan.rec_rr, gan.rec_iters = 3, 2
    x = torch.tensor(O.synthetic_images("mnist", gan.weights, 5)).cuda()
    z0 = torch.tensor(O.sample_z0(15, 128)).cuda()
    assert torch.equal(reconstruct_sharded(gan, x, z_init_val=z0), gan.reconstruct(x, z_init_val=z0))
    # z0 statistics through the public path: L=1 returns G(z0) of the best restart; use the generator's Linear
    # pre-activation scale as a proxy is overkill - check instead that two seeds differ and a seed repeats
    nat = gan._get_native(x.device)
    a = nat.reconstruct(x, 3, 1, 10.0, seed=123)
    b = nat.reconstruct(x, 3, 1, 10.0, seed=123)
    c_ = nat.reconstruct(x, 3, 1, 10.0, seed=124)
    assert torch.equal(a, b) and not torch.equal(a, c_)
    gan.close()


def _model_a_like(seed=0):
    """Random-weight stand-in for the reference's classifier A (utils/network_builder.py:412-427:
    conv 64 5x5 s1 -> relu -> conv 64 5x5 s2 -> relu -> flatten -> dense 128 -> relu -> dense 10)."""
    torch.manual_seed(seed)
    return torch.nn.Sequential(
        torch.nn.Conv2d(1, 64, 5, padding=2), torch.nn.ReLU(), torch.nn.Conv2d(64, 64, 5, stride=2), torch.nn.ReLU(),
        torch.nn.Flatten(), torch.nn.Linear(64 * 12 * 12, 128), torch.nn.ReLU(), torch.nn.Linear(128, 10)).eval()


def test_full_size_fp16_vs_fp32_and_classifier_agreement(gens):
    """BASELINE configs[1] operating point (MNIST, B=256, R=10, L=200): the fp16 tensor-core path against the
    fp32 CUDA-core path (which is oracle-checked elementwise at the sizes the CPU oracle can run):
    per-image |MSE_min difference| <= 1e-4 (BASELINE.json's bar), restart agreement and downstream
    classifier arg-max agreement reported (SURVEY 8d)."""
    arch = "mnist"
    w, gen16 = gens(arch, "fp16")
    _, gen32 = gens(arch, "fp32")
    B, R, L = 256, 10, 200
    x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
    z0 = torch.tensor(O.sample_z0(B * R, 128)).cuda()
    rec16, loss16, idx16 = gen16.reconstruct(x, R, L, 10.0, z_init_val=z0, return_aux=True)
    rec32, loss32, idx32 = gen32.reconstruct(x, R, L, 10.0, z_init_val=z0, return_aux=True)
    dmse = (loss16 - loss32).abs()
    agree = float((idx16 == idx32).float().mean())
    clf = _model_a_like().cuda()
    with torch.no_grad():
        p16 = clf(rec16.permute(0, 3, 1, 2)).argmax(1)
        p32 = clf(rec32.permute(0, 3, 1, 2)).argmax(1)
    cls_agree = float((p16 == p32).float().mean())
    print("C2 fp16 vs fp32: max|dMSE|=%.3g mean=%.3g restart agreement=%.3f classifier agreement=%.3f" % (
        float(dmse.max()), float(dmse.mean()), agree, cls_agree))
    assert float(dmse.max()) <= 1e-4
    assert agree >= 0.9 and cls_agree >= 0.97
    assert float(loss16.mean()) < 0.02            # the projection converged (targets are on-manifold + noise)
