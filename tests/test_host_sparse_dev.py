"""CPU tests (no GPU) of the sparse deviations (dgan_reconstruct[_measured[_csr / _conv]]_sparse_dev): the refusals of
the C entries and of Python before any native call, the binding's routing (None keeps today's entry), DefenseGANBase's
rec_sparse_dev, the cache name and its parse-back, the sharded call's refusal, and the fp64 oracle against autograd and
the closed form at step = 1."""
import ctypes
import os

import numpy as np
import pytest
import torch

from recording import Out, cpu_native, recording_gan  # noqa: F401  (the fixture)


INF = float("inf")
BAD = [(-1e-3, 1.0), (0.1, -1.0), (float("nan"), 1.0), (0.1, float("nan")), (INF, 1.0), (0.1, INF), (1e39, 1.0),
       (0.1, 1e39)]


# ---- refusals ----

def _entries(lib, sd):
    """Each entry without a handle, with sparse_dev sd: the counterpart's NULL check fails first."""
    return [lambda: lib.dgan_reconstruct_sparse_dev(None, None, None, None, None, None, 0, sd, None, None, None, None,
                                                    None, None, None, None, 0, None),
            lambda: lib.dgan_reconstruct_measured_sparse_dev(None, None, None, None, None, None, 0, sd, None, None, 10,
                                                             None, None, None, None, None, None, 0, None),
            lambda: lib.dgan_reconstruct_measured_csr_sparse_dev(None, None, None, None, None, None, 0, sd, None, None,
                                                                 None, None, 10, 5, None, None, None, None, None, None, 0,
                                                                 None),
            lambda: lib.dgan_reconstruct_measured_conv_sparse_dev(None, None, None, None, None, None, 0, sd, None, None,
                                                                  None, None, None, None, None, None, None, 0, None)]


@pytest.mark.parametrize("l1,step", BAD + [(0.0, 0.0), (0.1, 1.0)])
def test_c_entries_run_the_counterparts_checks_first(l1, step):
    from defensegan_b200 import _native
    lib = _native.load_library()
    sd = ctypes.byref(_native.dgan_sparse_dev(l1, step))
    for call in _entries(lib, sd) + _entries(lib, None):
        assert call() == -1
        assert lib.dgan_last_error().decode() == "NULL argument"
    assert lib.dgan_workspace_bytes_sparse_dev(None, 2, 2, 0, 0, None, 0) == 0


@pytest.mark.parametrize("l1,step", BAD)
def test_check_sparse_dev_names_the_bad_value(l1, step):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match="sparse_dev (l1|step)"):
        _native.check_sparse_dev((l1, step))


@pytest.mark.parametrize("bad", [None, 0.1, (0.1,), (0.1, 1.0, 2.0), (True, 1.0), ("0.1", 1.0)])
def test_check_sparse_dev_wants_a_pair_of_numbers(bad):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match="sparse_dev"):
        _native.check_sparse_dev(bad)


def test_check_sparse_dev_rounds_to_fp32_and_checks_eta_and_tau():
    from defensegan_b200 import _native
    assert _native.check_sparse_dev((0, 0)) == (0.0, 0.0)
    assert _native.check_sparse_dev((np.float64(0.1), 1)) == (float(np.float32(0.1)), 1.0)
    big = float(np.finfo(np.float32).max)
    assert _native.check_sparse_dev((0.1, big)) == (float(np.float32(0.1)), big)     # no n: eta unchecked
    with pytest.raises(ValueError, match="eta"):
        _native.check_sparse_dev((0.1, big), 784)
    with pytest.raises(ValueError, match="tau"):
        _native.check_sparse_dev((big, 1.0), 784)
    assert _native.check_sparse_dev((1.0, 1.0), 784) == (1.0, 1.0)


# ---- the binding's routing ----

def _obj(byref):
    return None if byref is None else byref._obj


def test_binding_routes_every_call_to_the_sparse_dev_entries(cpu_native):  # noqa: F811
    from defensegan_b200.operators import ConvOperator
    x = torch.rand(3, 28, 28, 1)
    pw = torch.ones(3, 28, 28, 1)
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 1.0
    cpu_native.reconstruct(x, 4, 9, 0.5, sparse_dev=(0.01, 1.0), out=Out(3 * 784))
    cpu_native.reconstruct(x, 4, 9, 0.01, adam=(0.8, 0.99, 1e-6), pixel_weights=pw, prune=[(2, 3)], huber_delta=0.5,
                           z_prior=0.1, sparse_dev=(0.0, 0.5), out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a, 4, 9, 1.0, sparse_dev=(0.2, 1.0), out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a.to_sparse_csr(), 4, 9, 1.0, prune=[(3, 2)],
                                    sparse_dev=(0.2, 1.0), out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 49), ConvOperator.box(4), 4, 9, 1.0, z_prior=0.5,
                                    sparse_dev=(0.3, 2.0), out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_sparse_dev", "dgan_reconstruct_sparse_dev"] * 2 + [
        "dgan_workspace_bytes_measured_sparse_dev", "dgan_reconstruct_measured_sparse_dev",
        "dgan_workspace_bytes_measured_sparse_dev", "dgan_reconstruct_measured_csr_sparse_dev",
        "dgan_workspace_bytes_measured_sparse_dev", "dgan_reconstruct_measured_conv_sparse_dev"]
    c = [args for _, args in cpu_native.calls]
    assert c[0][3] == 0 and c[0][4] == 0 and c[0][6] == 0                   # unweighted, momentum, unpruned
    assert c[1][2] is None and c[1][3] is None and c[1][4] is None and c[1][6] == 0
    sd = _obj(c[1][7])
    assert (sd.l1, sd.step) == (pytest.approx(0.01), 1.0) and c[1][8].value is None and c[1][10].value is None
    assert c[2][3] == 1 and c[2][4] == 1 and c[2][6] == 1                   # weighted, Adam, one prune point
    assert _obj(c[3][3]).value == 0.5 and _obj(c[3][4]).value == pytest.approx(0.1) and c[3][10].value is not None
    assert c[4][3:6] == (10, -1, None) and c[5][10] == 10
    assert c[6][3:5] == (10, 10) and c[7][6] == 1 and c[7][12:14] == (10, 10)
    assert c[8][3] == 49 and _obj(c[8][5]).kh == 4 and _obj(c[9][4]).value == 0.5 and _obj(c[9][9]).stride == 4


def test_binding_without_sparse_dev_routes_exactly_as_before(cpu_native):  # noqa: F811
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    cpu_native.reconstruct(x, 2, 5, out=Out(3 * 784))
    cpu_native.reconstruct(x, 2, 5, sparse_dev=None, deviation_out=None, z_prior=0.1, out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, sparse_dev=None, out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a.to_sparse_csr(), 2, 5, sparse_dev=None, out=Out(3 * 784))
    assert [c[0] for c in cpu_native.calls] == [
        "dgan_workspace_bytes", "dgan_reconstruct", "dgan_workspace_bytes", "dgan_reconstruct_prior",
        "dgan_workspace_bytes_measured", "dgan_reconstruct_measured", "dgan_workspace_bytes_measured_csr",
        "dgan_reconstruct_measured_csr"]


def test_binding_refuses_bad_arguments_before_any_native_call(cpu_native):  # noqa: F811
    from defensegan_b200.operators import ConvOperator
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    for bad in BAD:
        with pytest.raises(ValueError, match="sparse_dev"):
            cpu_native.reconstruct(x, 2, 5, sparse_dev=bad)
        with pytest.raises(ValueError, match="sparse_dev"):
            cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, sparse_dev=bad)
        with pytest.raises(ValueError, match="sparse_dev"):
            cpu_native.reconstruct_measured(torch.rand(3, 49), ConvOperator.box(4), 2, 5, sparse_dev=bad)
    with pytest.raises(ValueError, match="eta"):
        cpu_native.reconstruct(x, 2, 5, sparse_dev=(0.0, 1e36))
    with pytest.raises(ValueError, match="deviation_out needs sparse_dev"):
        cpu_native.reconstruct(x, 2, 5, deviation_out=torch.zeros(3, 28, 28, 1))
    with pytest.raises(ValueError, match="deviation_out must be"):
        cpu_native.reconstruct(x, 2, 5, sparse_dev=(0.1, 1.0), deviation_out=torch.zeros(3, 28, 28, 1))   # not CUDA
    with pytest.raises(ValueError, match="deviation_out must be"):
        cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, sparse_dev=(0.1, 1.0), deviation_out=Out(5))
    assert cpu_native.calls == []


# ---- DefenseGANBase ----

def test_defaults_cfg_key_and_kwargs():
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.operators import ConvOperator
    from defensegan_b200.utils.config import load_config, packaged_cfg_path
    assert MnistDefenseGAN(test_mode=True, verbose=False).rec_sparse_dev is None
    cfg = dict(load_config(packaged_cfg_path("mnist")))
    cfg["REC_SPARSE_DEV"] = [0.01, 1.0]
    assert MnistDefenseGAN(cfg=cfg, test_mode=True, verbose=False).rec_sparse_dev == [0.01, 1.0]
    gan, seen = recording_gan()
    a = torch.eye(784)[:10]
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    assert "sparse_dev" not in seen[0][1] and "deviation_out" not in seen[0][1] and "sparse_dev" not in seen[1][1]
    gan.rec_sparse_dev = (0.02, 1)
    dev = torch.zeros(2, 28, 28, 1)
    gan.reconstruct(torch.rand(2, 28, 28, 1), deviation_out=dev)
    gan.reconstruct_measured(torch.rand(2, 10), a.to_sparse_csr())
    gan.reconstruct_measured(torch.rand(2, 49), ConvOperator.box(4), deviation_out=dev)
    for _, kw in seen[2:]:
        assert kw["sparse_dev"] == (pytest.approx(0.02), 1.0)
    assert seen[2][1]["deviation_out"] is dev and seen[3][1]["deviation_out"] is None and seen[4][1]["deviation_out"] is dev


@pytest.mark.parametrize("val", [(-0.5, 1.0), (0.1, float("nan")), (INF, 1.0), 0.1, "x"])
def test_bad_rec_sparse_dev_is_refused_before_any_native_call(val):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    gan.rec_sparse_dev = val
    with pytest.raises(ValueError, match="rec_sparse_dev"):
        gan.reconstruct(torch.rand(2, 28, 28, 1))
    with pytest.raises(ValueError, match="rec_sparse_dev"):
        gan.reconstruct_measured(torch.rand(2, 10), torch.eye(784)[:10])
    with pytest.raises(ValueError, match="rec_sparse_dev"):
        gan.rec_cache_dir("test")
    gan.rec_sparse_dev = None
    with pytest.raises(ValueError, match="deviation_out needs rec_sparse_dev"):
        gan.reconstruct(torch.rand(2, 28, 28, 1), deviation_out=torch.zeros(2, 28, 28, 1))


def test_rec_cache_dir_names_sparse_dev_and_parses_back(tmp_path):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils import experiment as E
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 10.0, 200
    plain = gan.rec_cache_dir("test")
    assert "_sdev" not in plain
    gan.rec_sparse_dev = (0.01, 1.0)
    sd = gan.rec_cache_dir("test")
    assert sd.endswith(os.path.join("recs_rr10_lr10.00000_iters200_sdev0.01_1", "test"))
    gan.rec_huber_delta, gan.rec_z_prior, gan.rec_sparse_dev = 0.5, 0.1, (2.5e-05, 0.5)
    both = gan.rec_cache_dir("dev", max_num=100)
    assert both.endswith(os.path.join("recs_rr10_lr10.00000_iters200_num100_huber0.5_zprior0.1_sdev2.5e-05_0.5", "dev"))

    def parsed(path):
        other = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
        other.rec_sparse_dev = (7.0, 7.0)                    # overwritten by whatever the name says
        E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=path, override=False,
                                                  online_training=False, train_on_recs=False))
        return other

    assert parsed(plain).rec_sparse_dev is None
    assert parsed(sd).rec_sparse_dev == (pytest.approx(0.01), 1.0)
    other = parsed(both)
    assert other.rec_sparse_dev == (pytest.approx(2.5e-05), 0.5) and other.rec_z_prior == pytest.approx(0.1)
    for path in (plain, sd, both):
        assert parsed(path).rec_cache_dir(os.path.basename(path), max_num=100 if "num100" in path else -1) == path


def test_reconstruct_sharded_refuses_sparse_dev():
    from defensegan_b200 import parallel
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    gan.rec_sparse_dev = (0.01, 1.0)
    with pytest.raises(RuntimeError, match="rec_sparse_dev"):
        parallel.reconstruct_sharded(gan, torch.rand(2, 28, 28, 1))


# ---- the oracle ----

def _setup(b=2, rr=3, seed=0):
    from oracle import defensegan_oracle as O
    weights = O.init_generator_weights("mnist", seed=seed, latent_dim=16, net_dim=16, random_bias=True)
    x = np.random.RandomState(seed).uniform(0.0, 1.0, (b, 28, 28, 1)).astype(np.float32)
    z0 = O.sample_z0(b * rr, 16, 7)
    return weights, x, z0


@pytest.mark.parametrize("case", ["image", "weighted_huber", "measured"])
def test_oracle_matches_autograd_on_a_tiny_generator(case):
    """Two iterations of the oracle against an independent torch-autograd loop on J(z, nu) itself: the gradient of J in
    z and the proximal step on nu, from the same z0."""
    import huber_oracle as H
    import measured_oracle as MO
    import sparse_dev_oracle as S
    from oracle import defensegan_oracle as O
    weights, x, z0 = _setup()
    rr, l1, step, lam, lr = 3, 2e-4, 0.7, 0.05, 0.5
    kw = dict(images=x)
    if case == "weighted_huber":
        kw.update(pixel_weights=np.random.RandomState(4).uniform(0, 1, x.shape).astype(np.float32), delta=0.1)
    if case == "measured":
        a = MO.gaussian_operator(40, 784, seed=1)
        kw = dict(operator=a, measurements=np.random.RandomState(3).standard_normal((2, 40)).astype(np.float32) * 0.3)
    got = S.reconstruct("mnist", weights, rr, 3, lr, l1, step, lam=lam, z_init_val=z0, **kw)
    p = H._Problem("mnist", weights, rr, kw.get("delta", INF), kw.get("images"), kw.get("pixel_weights"),
                   kw.get("operator"), kw.get("measurements"))
    n = 40 if case == "measured" else 784
    l1f, stepf, lamf = (float(np.float32(v)) for v in (l1, step, lam))
    eta = stepf * n / 2
    z = torch.tensor(z0, dtype=torch.float64)
    nu = torch.zeros(z.shape[0], 784, dtype=torch.float64)
    v = torch.zeros_like(z)
    for t in range(3):
        zt, nt = z.clone().requires_grad_(True), nu.clone().requires_grad_(True)
        y = O.generator_forward("mnist", p.w, zt)
        u = y.reshape(y.shape[0], -1) + nt
        if p.a is not None:
            d = H.measured_loss(u, p.a, p.target, p.delta)
        else:
            d = H.image_loss(u.reshape(p.target.shape), p.target, p.delta, p.pw)
        smooth = d + lamf * (zt * zt).sum(dim=1)
        j = smooth + l1f * nt.abs().sum(dim=1)
        if t == 2:
            break
        gz, gn = torch.autograd.grad(smooth.sum(), (zt, nt))
        v = 0.7 * v + gz
        z = z - lr * v
        a_ = nu - eta * gn
        nu = torch.where(a_.abs() > eta * l1f, a_ - torch.sign(a_) * eta * l1f, torch.zeros_like(a_))
    assert np.allclose(got["loss_all"], j.detach().numpy(), rtol=1e-12, atol=1e-15)
    assert np.allclose(got["nu_all"], nu.numpy(), rtol=1e-12, atol=1e-15)
    assert np.allclose(got["z_final"], z.numpy(), rtol=1e-12, atol=1e-15)


def test_oracle_step_one_is_the_closed_form():
    """At step = 1 on the unweighted squared error the first nu step is S_tau(x - G(z0)) with tau = l1 n / 2, and J at
    L = 1 is D + l1 ||0||_1 = D."""
    import sparse_dev_oracle as S
    from oracle import defensegan_oracle as O
    weights, x, z0 = _setup()
    rr, l1 = 3, 1e-4
    r2 = S.reconstruct("mnist", weights, rr, 2, 0.0, l1, 1.0, images=x, z_init_val=z0)
    w = O.weights_to_torch(weights, torch.float64)
    g0 = O.generator_forward("mnist", w, torch.tensor(z0, dtype=torch.float64)).reshape(len(z0), -1)
    xt = torch.tensor(x, dtype=torch.float64).reshape(2, -1).repeat_interleave(rr, dim=0)
    tau = 784 / 2 * float(np.float32(l1))
    want = S.shrink(xt - g0, tau)
    assert float(want.abs().sum()) > 0 and float((want == 0).double().mean()) > 0.05     # both sides of the threshold
    assert np.allclose(r2["nu_all"], want.numpy(), rtol=1e-12, atol=1e-15)
    # rec_lr = 0 keeps z: J at iteration 1 is D at G(z0) + nu1 plus l1 ||nu1||_1
    d1 = ((g0 + want - xt) ** 2).mean(dim=1) + float(np.float32(l1)) * want.abs().sum(dim=1)
    assert np.allclose(r2["loss_all"], d1.numpy(), rtol=1e-12)
    r1 = S.reconstruct("mnist", weights, rr, 1, 0.0, l1, 1.0, images=x, z_init_val=z0)
    assert np.allclose(r1["loss_all"], ((g0 - xt) ** 2).mean(dim=1).numpy(), rtol=1e-12)


def test_oracle_at_step_zero_reproduces_the_prior_oracle():
    import prior_oracle as P
    import sparse_dev_oracle as S
    weights, x, z0 = _setup()
    r0 = P.reconstruct("mnist", weights, 3, 5, 1.0, 0.1, images=x, z_init_val=z0)
    r1 = S.reconstruct("mnist", weights, 3, 5, 1.0, 0.3, 0.0, lam=0.1, images=x, z_init_val=z0)
    for k in ("loss_all", "rec_all", "idx", "z_final"):
        assert np.allclose(r0[k], r1[k], rtol=1e-12, atol=1e-15), k
    assert not r1["nu_all"].any()
