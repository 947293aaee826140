"""Wider GPU parity evidence at the metric's operating point (R=10, L=200), through the C-ABI.

What each test pins (all `-m gpu`; the CPU oracle runs on the GPU box's host cores):
  * worst-case images (S2: i.i.d. uniform, far from the generator's range) for MNIST against the fp32 AND the fp64
    oracle, both precisions: per-image |MSE_min - oracle| <= 1e-4 (BASELINE.json's bar), margin printed;
  * on-manifold images (S1) at B=32 against the oracle;
  * CelebA (64x64x3, tanh, 4 deconvs) at R=10, L=200 against the oracle, and at BASELINE configs[3] size
    (B=128) fp16 against the fp32 CUDA path;
  * the Philox z0 initialiser: moments of N(0, 1/latent_dim) over 2^20 samples, tiling independence, and that a
    call with z_init_val=None starts from exactly that draw (models/gan.py:370-377);
  * ReconstructionLayer / add_rec_model (utils/network_builder.py:179-183,239-271);
  * decay_lr=1 (the evidently intended schedule) against the oracle's emulate_dead_decay=False;
  * large, saturating weights (trained-checkpoint-like magnitudes): finite results, fp16 close to the oracle;
  * 2 NCCL ranks == 1 GPU, bit for bit, with z_init_val given and with the shared Philox stream.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MSE_BAR = 1e-4     # BASELINE.json: "reconstruction MSE within 1e-4 of the reference"


def _native_gen(arch, weights, precision):
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    return _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in weights.values()], precision=precision,
                                   device=dev)


@pytest.fixture(scope="module")
def gens():
    cache = {}

    def get(arch, precision):
        if (arch, precision) not in cache:
            w = O.init_generator_weights(arch)
            cache[(arch, precision)] = (w, _native_gen(arch, w, precision))
        return cache[(arch, precision)]

    yield get
    for _, g in cache.values():
        g.close()


@pytest.fixture(scope="module")
def oracle_runs():
    """Oracle results shared by the two precisions of a test (the oracle is the slow part)."""
    cache = {}

    def get(arch, kind, B, R, L, dtype):
        key = (arch, kind, B, R, L, dtype)
        if key not in cache:
            torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
            w = O.init_generator_weights(arch)
            imgs = O.synthetic_images(arch, w, B, kind=kind)
            z0 = O.sample_z0(B * R, 128)
            cache[key] = (imgs, z0, O.reconstruct(arch, w, imgs, R, L, z_init_val=z0, dtype=dtype))
        return cache[key]

    return get


def _run(gen, imgs, z0, R, L, **kw):
    rec, loss, idx = gen.reconstruct(torch.tensor(imgs).cuda(), R, L, 10.0, z_init_val=torch.tensor(z0).cuda(),
                                     return_aux=True, **kw)
    return rec.cpu().numpy(), loss.cpu().numpy(), idx.cpu().numpy()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_mnist_worst_case_images_l200_vs_fp32_and_fp64_oracle(gens, oracle_runs, precision):
    """S2 targets never get close to the generator's range, so all R restarts keep moving for all 200 steps and rounding
    differences have the longest lever; the oracle's own fp32-vs-fp64 drift is printed next to ours."""
    arch, B, R, L = "mnist", 16, 10, 200
    imgs, z0, r32 = oracle_runs(arch, "S2", B, R, L, torch.float32)
    _, _, r64 = oracle_runs(arch, "S2", B, R, L, torch.float64)
    _, gen = gens(arch, precision)
    rec, loss, idx = _run(gen, imgs, z0, R, L)
    d32, d64 = np.abs(loss - r32["loss_min"]), np.abs(loss - r64["loss_min"])
    drift = np.abs(r32["loss_min"] - r64["loss_min"])
    print("S2 mnist L=200 %s: max|dMSE| vs fp32 oracle %.3g, vs fp64 oracle %.3g (oracle fp32-vs-fp64 %.3g); margin to "
          "1e-4: x%.1f; restart agreement %.2f / %.2f" % (precision, d32.max(), d64.max(), drift.max(),
                                                          MSE_BAR / max(d32.max(), d64.max(), 1e-12),
                                                          (idx == r32["idx"]).mean(), (idx == r64["idx"]).mean()))
    assert np.isfinite(rec).all()
    assert d32.max() <= MSE_BAR and d64.max() <= MSE_BAR


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_mnist_on_manifold_l200_b32_vs_oracle(gens, oracle_runs, precision):
    arch, B, R, L = "mnist", 32, 10, 200
    imgs, z0, r32 = oracle_runs(arch, "S1", B, R, L, torch.float32)
    _, gen = gens(arch, precision)
    rec, loss, idx = _run(gen, imgs, z0, R, L)
    d = np.abs(loss - r32["loss_min"])
    print("S1 mnist L=200 B=32 %s: max|dMSE| %.3g mean %.3g restart agreement %.2f" % (precision, d.max(), d.mean(),
                                                                                    (idx == r32["idx"]).mean()))
    assert d.max() <= MSE_BAR
    # the chosen reconstructions themselves: where the same restart won, pixels agree to fp16-forward accuracy
    same = idx == r32["idx"]
    assert same.mean() >= 0.8
    assert np.abs(rec[same] - r32["rec"][same]).max() <= (2e-2 if precision == "fp16" else 5e-3)


@pytest.mark.parametrize("kind", ["S1", "S2"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_celeba_l200_vs_oracle(gens, oracle_runs, precision, kind):
    """BASELINE configs[3] operating point (R=10, L=200) on a batch the oracle finishes quickly."""
    arch, B, R, L = "celeba", 4, 10, 200
    imgs, z0, r32 = oracle_runs(arch, kind, B, R, L, torch.float32)
    _, gen = gens(arch, precision)
    rec, loss, idx = _run(gen, imgs, z0, R, L)
    d = np.abs(loss - r32["loss_min"])
    print("%s celeba L=200 %s: max|dMSE| %.3g (loss ~%.3g) restart agreement %.2f" % (kind, precision, d.max(),
                                                                                      r32["loss_min"].mean(),
                                                                                      (idx == r32["idx"]).mean()))
    assert np.isfinite(rec).all()
    assert d.max() <= MSE_BAR


def test_celeba_full_size_fp16_vs_fp32(gens):
    """BASELINE configs[3]: CelebA B=128, R=10, L=200 - the tensor-core path against the fp32 CUDA-core path (which the
    test above pins to the oracle)."""
    arch, B, R, L = "celeba", 128, 10, 200
    w, g16 = gens(arch, "fp16")
    _, g32 = gens(arch, "fp32")
    imgs = O.synthetic_images(arch, w, B)
    z0 = O.sample_z0(B * R, 128)
    rec16, l16, i16 = _run(g16, imgs, z0, R, L)
    rec32, l32, i32 = _run(g32, imgs, z0, R, L)
    d = np.abs(l16 - l32)
    print("C4 celeba fp16 vs fp32: max|dMSE| %.3g mean %.3g restart agreement %.3f" % (d.max(), d.mean(), (i16 == i32).mean()))
    assert d.max() <= MSE_BAR
    assert (i16 == i32).mean() >= 0.9


def test_philox_z0_statistics_and_tiling(gens):
    """z_hat ~ N(0, 1/latent_dim) i.i.d. (models/gan.py:370-377): first four moments over 2^20 samples, independence of
    how the rows are tiled (the counter is the global element index), and that the projection really starts there."""
    w, gen = gens("mnist", "fp32")
    n_rows, latent = 8192, 128
    z = gen.sample_z0(n_rows, seed=20240917).double()
    n = z.numel()
    sigma2 = 1.0 / latent
    mean, var = float(z.mean()), float(z.var(unbiased=False))
    zs = z / sigma2 ** 0.5
    skew, kurt = float((zs ** 3).mean()), float((zs ** 4).mean()) - 3.0
    print("Philox z0: n=%d mean %.3g (sigma/sqrt(n) %.3g) var*latent %.5f skew %.4f excess kurtosis %.4f" % (
        n, mean, (sigma2 / n) ** 0.5, var * latent, skew, kurt))
    assert abs(mean) <= 5.0 * (sigma2 / n) ** 0.5
    assert abs(var / sigma2 - 1.0) <= 5.0 * (2.0 / n) ** 0.5          # sd of the sample variance of a normal
    assert abs(skew) <= 5.0 * (6.0 / n) ** 0.5 and abs(kurt) <= 5.0 * (24.0 / n) ** 0.5
    # no obvious dependence: rows/columns uncorrelated, |z| tail mass as a normal's
    assert abs(float((zs[:, :-1] * zs[:, 1:]).mean())) <= 5.0 / (n ** 0.5)
    assert abs(float((zs[:-1] * zs[1:]).mean())) <= 5.0 / (n ** 0.5)
    tail = float((zs.abs() > 3.0).double().mean())
    assert abs(tail - 0.0026998) <= 5.0 * (0.0027 / n) ** 0.5
    # tiling independence: any window of rows equals the same rows of the big draw; another seed differs
    sub = gen.sample_z0(100, seed=20240917, z_row_offset=1234)
    assert torch.equal(sub.double(), z[1234:1334])
    assert not torch.equal(gen.sample_z0(100, seed=20240918, z_row_offset=1234).double(), z[1234:1334])
    # the loop starts from exactly this draw
    B, R = 6, 4
    x = torch.tensor(O.synthetic_images("mnist", w, B)).cuda()
    a = gen.reconstruct(x, R, 3, 10.0, seed=77, return_aux=True)
    b = gen.reconstruct(x, R, 3, 10.0, z_init_val=gen.sample_z0(B * R, seed=77), return_aux=True)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    # and a shard of the batch with its row offset reproduces the corresponding rows
    c = gen.reconstruct(x[2:], R, 3, 10.0, seed=77, z_row_offset=2 * R, return_aux=True)
    assert torch.equal(c[0], a[0][2:]) and torch.equal(c[1], a[1][2:]) and torch.equal(c[2], a[2][2:])


def test_reconstruction_layer_and_add_rec_model():
    """utils/network_builder.py:239-271: fprop(x) = gan.reconstruct(x, batch_size, back_prop, reconstructor_id=123,
    z_init_val); :179-183: add_rec_model puts it in front of the classifier."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils.network_builder import ReconstructionLayer, add_rec_model
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp16")
    gan.rec_rr, gan.rec_iters = 3, 6
    B = 5
    x = torch.tensor(O.synthetic_images("mnist", gan.weights, B)).cuda()
    z0 = torch.tensor(O.sample_z0(B * 3, 128)).cuda()
    layer = ReconstructionLayer(gan, [None, 28, 28, 1], B, z_init_val=z0)
    assert layer.get_output_shape() == [None, 28, 28, 1]
    want = gan.reconstruct(x, batch_size=B, reconstructor_id=123, z_init_val=z0)
    assert torch.equal(layer.fprop(x), want)
    assert torch.equal(layer.fprop(x.reshape(B, 784)), want)            # fprop reshapes to the input shape first
    # without z_init_val the layer draws with reconstructor_id 123: same counter state -> same draw as a direct call
    gan2 = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp16")
    gan2.rec_rr, gan2.rec_iters = 3, 6
    free = ReconstructionLayer(gan, [None, 28, 28, 1], B)
    gan._call_counter = gan2._call_counter = 0
    assert torch.equal(free.fprop(x), gan2.reconstruct(x, reconstructor_id=123))
    torch.manual_seed(0)
    clf = torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(784, 10)).cuda()
    model = add_rec_model(clf, gan, [None, 28, 28, 1], batch_size=B, z_init_val=z0)
    with torch.no_grad():
        assert torch.equal(model(x), clf(want))
        assert torch.equal(model.get_probs(x), clf(want))
    gan.close()
    gan2.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_intended_lr_decay_option(gens, precision):
    """decay_lr=1: lr x0.1 from step ceil(0.8 L) (base_model.py:153-194 as evidently intended; off by default because
    the reference's schedule never advances, SURVEY F3)."""
    arch, B, R, L = "mnist", 6, 3, 30
    w, gen = gens(arch, precision)
    imgs = O.synthetic_images(arch, w, B, kind="S2", seed=11)
    z0 = O.sample_z0(B * R, 128, seed=12)
    want = O.reconstruct(arch, w, imgs, R, L, z_init_val=z0, emulate_dead_decay=False)
    const = O.reconstruct(arch, w, imgs, R, L, z_init_val=z0)
    gap = float(np.abs(want["loss_min"] - const["loss_min"]).min())
    assert gap > 1e-5                                             # the option changes every image's result ...
    rec, loss, idx = _run(gen, imgs, z0, R, L, decay_lr=True)
    rec_c, loss_c, _ = _run(gen, imgs, z0, R, L)
    err_d, err_c = np.abs(loss - want["loss_min"]).max(), np.abs(loss_c - const["loss_min"]).max()
    print("decay_lr %s: |decayed - oracle| %.3g, |constant - oracle| %.3g, decayed-vs-constant gap %.3g" % (precision, err_d, err_c, gap))
    # ... and each run sits much closer to its own oracle than the two schedules are apart
    assert err_d <= 0.25 * gap and err_c <= 0.25 * gap
    assert np.abs(loss - const["loss_min"]).min() >= 0.5 * gap


def test_large_saturating_weights_stay_finite(gens):
    """Trained checkpoints have larger filters than He-init: scale every filter x3 and add biases so that the sigmoid
    saturates and backward activations grow; the fp16 path must stay finite (saturating fp16 conversion) and close to
    the fp32 oracle at a short horizon."""
    arch, B, R, L = "mnist", 8, 4, 30
    w = O.init_generator_weights(arch, random_bias=True)
    big = {k: (v * 3.0 if k.endswith(".Filters") or k.endswith(".W") else v) for k, v in w.items()}
    imgs = O.synthetic_images(arch, w, B, kind="S2", seed=3)
    z0 = O.sample_z0(B * R, 128, seed=4)
    want = O.reconstruct(arch, big, imgs, R, L, rec_lr=1.0, z_init_val=z0)
    for precision, tol in (("fp32", 2e-4), ("fp16", 5e-3)):
        gen = _native_gen(arch, big, precision)
        rec, loss, idx = gen.reconstruct(torch.tensor(imgs).cuda(), R, L, 1.0, z_init_val=torch.tensor(z0).cuda(), return_aux=True)
        assert torch.isfinite(rec).all() and torch.isfinite(loss).all()
        d = np.abs(loss.cpu().numpy() - want["loss_min"])
        print("x3 weights %s: max|dMSE| %.3g (loss ~%.3g)" % (precision, d.max(), want["loss_min"].mean()))
        assert d.max() <= tol
        gen.close()


def test_reconstruct_dataset_real_projector_and_cache(tmp_path):
    """f1 (models/gan.py:451-587) with the real projector: a 2-batch synthetic split is reconstructed, cached per image
    and as feats.pkl, and a second pass is served from the cache without touching the GPU path."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp16", output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_iters = 2, 4
    gan.initialized = True                                      # keep the random-init generator
    raw = (O.synthetic_images("mnist", gan.weights, 6) * 255.0).astype("float32")
    labels = np.arange(6) % 10

    def split():
        return [(raw[0:3], labels[0:3]), (raw[3:6], labels[3:6])]

    gan.set_dataset_generators(train=split, dev=split, test=split)
    rets = gan.reconstruct_dataset()
    recs, tgts, orig = rets["test"]
    assert recs.shape == (6, 28, 28, 1) and orig.shape == (6, 28, 28, 1) and list(tgts) == list(labels)
    assert np.allclose(orig, raw / 255.0)
    mse = ((recs - orig) ** 2).mean(axis=(1, 2, 3))
    assert np.all(np.isfinite(recs)) and float(mse.mean()) < float(((0.5 - orig) ** 2).mean())
    d = gan.rec_cache_dir("test")
    assert os.path.isfile(os.path.join(d, "pickles", "rec_0000004_l4.pkl"))
    calls = []
    real = gan.reconstruct
    gan.reconstruct = lambda *a, **k: calls.append(1) or real(*a, **k)
    again = gan.reconstruct_dataset()
    assert not calls                                            # every batch came from the per-image cache
    assert np.array_equal(again["test"][0], recs)
    gan.save_recs(rets)
    third = gan.reconstruct_dataset()
    assert not calls and np.array_equal(third["train"][0], rets["train"][0])
    gan.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_nccl_ranks_equal_one_gpu(tmp_path):
    """SURVEY section 4(v): the sharded result gathered over NCCL == the single-GPU result, bit for bit, on the real
    kernels - with z_init_val given and with the shared Philox stream (z_init_val=None)."""
    out = tmp_path / "nccl.json"
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29613", os.path.join(ROOT, "tests", "nccl_worker.py"), str(out)]
    res = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-4000:]
    import json
    r = json.loads(out.read_text())
    assert r["equal_given_z0"] and r["equal_random_z0"] and r["equal_ragged"], r
