"""CPU tests (no GPU) of the latent prior (dgan_reconstruct_prior, dgan_reconstruct_measured[_csr / _conv]_prior): the
refusal of a bad lambda by the C entries and by Python before any native call, the binding's routing (a call without the
prior keeps its entry and kwargs), DefenseGANBase's rec_z_prior, the cache name and its parse-back, and the prior oracle
against finite differences and the existing oracles."""
import ctypes
import os

import numpy as np
import pytest
import torch

from recording import Out, cpu_native, recording_gan  # noqa: F401  (the fixture)


INF = float("inf")
BAD = [-1e-3, -INF, INF, float("nan"), 3e38, 1e39]        # 3e38: finite in fp32, 2 lambda is not; 1e39: inf in fp32


# ---- refusals ----

def _entries(lib, lam, ap=None):
    """Each prior entry with lambda, Adam parameters ap (NULL: momentum) and NULL / 0 for the rest, but valid scalars
    where the counterpart checks them before the handle (m = 10, nnz = 5)."""
    return {
        "dgan_reconstruct_prior": lambda: lib.dgan_reconstruct_prior(None, None, ap, None, lam, None, 0, None, None, None,
                                                                     None, None, None, None, 0, None),
        "dgan_reconstruct_measured_prior": lambda: lib.dgan_reconstruct_measured_prior(
            None, None, ap, None, lam, None, 0, None, 10, None, None, None, None, None, None, 0, None),
        "dgan_reconstruct_measured_csr_prior": lambda: lib.dgan_reconstruct_measured_csr_prior(
            None, None, ap, None, lam, None, 0, None, None, None, 10, 5, None, None, None, None, None, None, 0, None),
        "dgan_reconstruct_measured_conv_prior": lambda: lib.dgan_reconstruct_measured_conv_prior(
            None, None, ap, None, lam, None, 0, None, None, None, None, None, None, None, None, 0, None)}


@pytest.mark.parametrize("lam", BAD + [0.0, 0.1])
def test_c_entries_run_the_counterparts_checks_first(lam):
    """Without a handle every entry fails the counterpart's NULL check, whatever lambda: lambda comes after it."""
    from defensegan_b200 import _native
    lib = _native.load_library()
    for sym, call in _entries(lib, lam).items():
        assert call() == -1, sym
        msg = lib.dgan_last_error().decode()
        assert msg in ("NULL argument", "invalid argument"), (sym, msg)
        bad_adam = ctypes.byref(_native.dgan_adam_params(1.0, 0.999, 1e-8))
        assert _entries(lib, lam, bad_adam)[sym]() == -1
        assert "invalid Adam parameters" in lib.dgan_last_error().decode(), sym


@pytest.mark.parametrize("bad", BAD + [True, "0.1", None, [0.1], -10 ** 400, 10 ** 400])
def test_check_z_prior_names_the_bad_value(bad):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match="z_prior"):
        _native.check_z_prior(bad)


def test_check_z_prior_accepts_finite_non_negative_values_as_fp32():
    from defensegan_b200 import _native
    assert _native.check_z_prior(0) == 0.0 and _native.check_z_prior(0.0) == 0.0
    assert _native.check_z_prior(np.float64(0.1)) == float(np.float32(0.1))
    assert _native.check_z_prior(2) == 2.0
    assert _native.check_z_prior(1e-50) == 0.0                      # rounds to 0 in fp32
    big = float(np.float32(np.finfo(np.float32).max) / np.float32(2))
    assert _native.check_z_prior(big) == big                        # 2 lambda is FLT_MAX


# ---- the binding's routing ----

def _obj(byref):
    return None if byref is None else byref._obj


def test_binding_routes_image_calls_to_the_prior_entry(cpu_native):  # noqa: F811
    x = torch.rand(3, 28, 28, 1)
    pw = torch.ones(3, 28, 28, 1)
    cpu_native.reconstruct(x, 4, 9, 0.5, seed=5, z_prior=0.25, out=Out(3 * 784))
    cpu_native.reconstruct(x, 4, 9, 0.01, adam=(0.8, 0.99, 1e-6), pixel_weights=pw, prune=[(2, 3)], huber_delta=0.5,
                           z_prior=0.0, out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes", "dgan_reconstruct_prior", "dgan_workspace_bytes_adam", "dgan_reconstruct_prior"]
    rc0, rc1 = cpu_native.calls[1][1], cpu_native.calls[3][1]
    assert rc0[2] is None and rc0[3] is None and rc0[4] == 0.25 and rc0[5] is None and rc0[6] == 0
    assert rc0[8].value is None                                    # w_dev NULL
    assert _obj(rc1[2]).beta1 == pytest.approx(0.8) and _obj(rc1[3]).value == 0.5 and rc1[4] == 0.0
    assert rc1[6] == 1 and rc1[8].value is not None


def test_binding_routes_measured_calls_to_the_prior_entries(cpu_native):  # noqa: F811
    from defensegan_b200.operators import ConvOperator
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 1.0
    y = torch.rand(3, 10)
    cpu_native.reconstruct_measured(y, a, 4, 9, 1.0, z_prior=0.1, out=Out(3 * 784))
    cpu_native.reconstruct_measured(y, a.to_sparse_csr(), 4, 9, 0.01, adam=(0.9, 0.999, 1e-8), prune=[(3, 2)],
                                    huber_delta=0.1, z_prior=2.0, out=Out(3 * 784))
    op = ConvOperator.box(4)
    cpu_native.reconstruct_measured(torch.rand(3, 49), op, 4, 9, 1.0, z_prior=0.5, out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_measured", "dgan_reconstruct_measured_prior",
                     "dgan_workspace_bytes_measured_adam", "dgan_reconstruct_measured_csr_prior",
                     "dgan_workspace_bytes_measured_conv", "dgan_reconstruct_measured_conv_prior"]
    rc0, rc1, rc2 = cpu_native.calls[1][1], cpu_native.calls[3][1], cpu_native.calls[5][1]
    assert rc0[2] is None and rc0[3] is None and rc0[4] == pytest.approx(0.1) and rc0[6] == 0 and rc0[8] == 10
    assert rc1[2] is not None and _obj(rc1[3]).value == pytest.approx(0.1) and rc1[4] == 2.0 and rc1[6] == 1
    assert rc1[10:12] == (10, 10)
    assert rc2[2] is None and rc2[3] is None and rc2[4] == 0.5 and rc2[6] == 0 and (_obj(rc2[7]).kh, _obj(rc2[7]).stride) == (4, 4)


def test_binding_without_the_prior_routes_exactly_as_before(cpu_native):  # noqa: F811
    from defensegan_b200.operators import ConvOperator
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    cpu_native.reconstruct(x, 2, 5, out=Out(3 * 784))
    cpu_native.reconstruct(x, 2, 5, z_prior=None, huber_delta=0.5, out=Out(3 * 784))
    cpu_native.reconstruct(x, 2, 5, z_prior=None, prune=[(2, 1)], adam=(0.9, 0.999, 1e-8), out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, z_prior=None, out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 10), a.to_sparse_csr(), 2, 5, z_prior=None, out=Out(3 * 784))
    cpu_native.reconstruct_measured(torch.rand(3, 49), ConvOperator.box(4), 2, 5, z_prior=None, out=Out(3 * 784))
    assert [c[0] for c in cpu_native.calls] == [
        "dgan_workspace_bytes", "dgan_reconstruct", "dgan_workspace_bytes", "dgan_reconstruct_huber",
        "dgan_workspace_bytes_adam", "dgan_reconstruct_adam", "dgan_workspace_bytes_measured", "dgan_reconstruct_measured",
        "dgan_workspace_bytes_measured_csr", "dgan_reconstruct_measured_csr", "dgan_workspace_bytes_measured_conv",
        "dgan_reconstruct_measured_conv"]


def test_binding_refuses_a_bad_lambda_before_any_native_call(cpu_native):  # noqa: F811
    from defensegan_b200.operators import ConvOperator
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    for bad in BAD:
        with pytest.raises(ValueError, match="z_prior"):
            cpu_native.reconstruct(x, 2, 5, z_prior=bad)
        with pytest.raises(ValueError, match="z_prior"):
            cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, z_prior=bad)
        with pytest.raises(ValueError, match="z_prior"):
            cpu_native.reconstruct_measured(torch.rand(3, 10), a.to_sparse_csr(), 2, 5, z_prior=bad)
        with pytest.raises(ValueError, match="z_prior"):
            cpu_native.reconstruct_measured(torch.rand(3, 49), ConvOperator.box(4), 2, 5, z_prior=bad)
    assert cpu_native.calls == []


# ---- DefenseGANBase ----

def test_defaults_and_cfg_key():
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils.config import load_config, packaged_cfg_path
    assert MnistDefenseGAN(test_mode=True, verbose=False).rec_z_prior is None
    cfg = dict(load_config(packaged_cfg_path("mnist")))
    cfg["REC_Z_PRIOR"] = 0.1
    assert MnistDefenseGAN(cfg=cfg, test_mode=True, verbose=False).rec_z_prior == 0.1


def test_calls_without_the_prior_keep_their_kwargs_and_prior_calls_add_lambda():
    from defensegan_b200.operators import ConvOperator
    gan, seen = recording_gan()
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10)] = 1.0
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    assert sorted(seen[0][1]) == ["decay_lr", "momentum", "out", "return_aux", "seed", "z_init_val", "z_row_offset"]
    assert "z_prior" not in seen[1][1]
    gan.rec_z_prior = 0.3
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    gan.reconstruct_measured(torch.rand(2, 10), a.to_sparse_csr(), prune=[(10, 2)])
    gan.reconstruct_measured(torch.rand(2, 49), ConvOperator.box(4))
    gan.rec_z_prior = 0
    gan.rec_huber_delta = 0.5
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    for _, kw in seen[2:6]:
        assert kw["z_prior"] == pytest.approx(0.3)
    assert seen[4][1]["prune"] == [(10, 2)]
    assert seen[6][1]["z_prior"] == 0.0 and seen[6][1]["huber_delta"] == 0.5


@pytest.mark.parametrize("val", [-0.5, float("nan"), INF, 1e39, "x"])
def test_bad_rec_z_prior_is_refused_before_any_native_call(val):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    gan.rec_z_prior = val
    with pytest.raises(ValueError, match="rec_z_prior"):
        gan.reconstruct(torch.rand(2, 28, 28, 1))
    with pytest.raises(ValueError, match="rec_z_prior"):
        gan.reconstruct_measured(torch.rand(2, 10), torch.eye(784)[:10])
    with pytest.raises(ValueError, match="rec_z_prior"):
        gan.rec_cache_dir("test")


def test_rec_cache_dir_names_lambda_and_parses_back(tmp_path):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils import experiment as E
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 10.0, 200
    plain = gan.rec_cache_dir("test")
    assert "_zprior" not in plain
    gan.rec_z_prior = 0.1
    pri = gan.rec_cache_dir("test")
    assert pri.endswith(os.path.join("recs_rr10_lr10.00000_iters200_zprior0.1", "test"))
    gan.rec_z_prior = 0
    zero = gan.rec_cache_dir("test")
    assert zero.endswith("_zprior0" + os.sep + "test")
    gan.rec_prune, gan.rec_optimizer, gan.rec_huber_delta, gan.rec_z_prior = [(40, 2)], "adam", 0.5, 2.5e-05
    both = gan.rec_cache_dir("dev", max_num=100)
    assert both.endswith(os.path.join(
        "recs_rr10_lr10.00000_iters200_num100_prune40x2_adam0.9-0.999-1e-08_huber0.5_zprior2.5e-05", "dev"))
    gan.rec_prune, gan.rec_optimizer, gan.rec_huber_delta, gan.rec_z_prior = None, "momentum", None, None
    assert gan.rec_cache_dir("test") == plain

    def parsed(path):
        other = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
        other.rec_z_prior = 7.0                             # overwritten by whatever the name says
        E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=path, override=False,
                                                  online_training=False, train_on_recs=False))
        return other

    assert parsed(plain).rec_z_prior is None
    assert parsed(pri).rec_z_prior == pytest.approx(0.1)
    assert parsed(zero).rec_z_prior == 0.0
    other = parsed(both)
    assert other.rec_z_prior == pytest.approx(2.5e-05) and other.rec_huber_delta == 0.5 and other.rec_optimizer == "adam"
    assert other.rec_cache_dir("dev", max_num=100) == both        # the parsed values name the same directory again
    for path in (plain, pri, zero, both):
        assert parsed(path).rec_cache_dir(os.path.basename(path), max_num=100 if "num100" in path else -1) == path


# ---- the oracle ----

def _setup(b=2, rr=3, seed=0):
    from oracle import defensegan_oracle as O
    weights = O.init_generator_weights("mnist", seed=seed, latent_dim=16, net_dim=16, random_bias=True)
    x = np.random.RandomState(seed).uniform(0.0, 1.0, (b, 28, 28, 1)).astype(np.float32)
    z0 = O.sample_z0(b * rr, 16, 7)
    return weights, x, z0


@pytest.mark.parametrize("case", ["image", "weighted", "huber", "measured"])
def test_oracle_gradient_of_j_matches_finite_differences(case):
    import measured_oracle as MO
    import prior_oracle as P
    weights, x, z0 = _setup()
    rr, lam = 3, 0.37
    kw = dict(images=x)
    if case == "weighted":
        kw["pixel_weights"] = np.random.RandomState(4).uniform(0, 1, x.shape).astype(np.float32)
    if case == "huber":
        kw["delta"] = 0.1
    if case == "measured":
        a = MO.gaussian_operator(40, 784, seed=1)
        kw = dict(operator=a, measurements=np.random.RandomState(3).standard_normal((2, 40)).astype(np.float32) * 0.3)
    _, d, j, g = P.loss_and_grad("mnist", weights, z0, rr, lam, **kw)
    z = z0.astype(np.float64)
    assert np.allclose(j - d, lam * (z * z).sum(axis=1), rtol=1e-12)
    _, _, _, g0 = P.loss_and_grad("mnist", weights, z0, rr, 0.0, **kw)
    assert np.allclose(g - g0, 2 * lam * z, rtol=1e-10, atol=1e-14)
    rng = np.random.RandomState(5)
    for _ in range(3):
        v = rng.standard_normal(z.shape)
        v /= np.linalg.norm(v)
        h = 1e-6
        jp = P.loss_and_grad("mnist", weights, z + h * v, rr, lam, **kw)[2].sum()
        jm = P.loss_and_grad("mnist", weights, z - h * v, rr, lam, **kw)[2].sum()
        assert (jp - jm) / (2 * h) == pytest.approx(float((g * v).sum()), rel=1e-5, abs=1e-9)


@pytest.mark.parametrize("adam", [None, (0.9, 0.999, 1e-8)])
def test_oracle_at_zero_reproduces_the_counterpart_oracles(adam):
    import huber_oracle as H
    import prior_oracle as P
    weights, x, z0 = _setup()
    lr = 0.05 if adam else 2.0
    r0 = H.reconstruct("mnist", weights, 3, 6, lr, INF, images=x, z_init_val=z0, adam=adam)
    r1 = P.reconstruct("mnist", weights, 3, 6, lr, 0.0, images=x, z_init_val=z0, adam=adam)
    for k in ("loss_all", "rec_all", "idx"):
        assert np.allclose(r0[k], r1[k], rtol=1e-12, atol=1e-14), k
    # a prior shrinks the chosen restarts' latents
    r2 = P.reconstruct("mnist", weights, 3, 6, lr, 0.5, images=x, z_init_val=z0, adam=adam)
    assert np.linalg.norm(r2["z_final"]) < np.linalg.norm(r1["z_final"])
