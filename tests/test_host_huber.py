"""CPU tests (no GPU) of the Huber data term (dgan_reconstruct_huber, dgan_reconstruct_measured[_csr]_huber,
dgan_loss_grad[_measured[_csr]]_huber): the refusal of a bad delta by the C entries and by Python before any native
call, the binding's routing (a squared-error call's entry and kwargs unchanged), DefenseGANBase's rec_huber_delta, the
cache name and its parse-back, and the Huber oracle against the existing oracles and finite differences."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from recording import Out, cpu_native, recording_gan  # noqa: F401  (the fixture)


BAD = [0.0, -0.0, -1.0, float("nan"), -float("inf"), 1e-50]       # 1e-50 is 0 in fp32


# ---- refusals ----

def _entries(lib, delta, ap=None):
    """Each Huber entry with delta, Adam parameters ap (NULL: momentum) and NULL / 0 for the rest, but valid scalars
    where the counterpart checks them before the handle (m = 10, nnz = 5)."""
    return {
        "dgan_reconstruct_huber": lambda: lib.dgan_reconstruct_huber(None, None, ap, delta, None, 0, None, None, None,
                                                                     None, None, None, None, 0, None),
        "dgan_reconstruct_measured_huber": lambda: lib.dgan_reconstruct_measured_huber(
            None, None, ap, delta, None, 0, None, 10, None, None, None, None, None, None, 0, None),
        "dgan_reconstruct_measured_csr_huber": lambda: lib.dgan_reconstruct_measured_csr_huber(
            None, None, ap, delta, None, 0, None, None, None, 10, 5, None, None, None, None, None, None, 0, None),
        "dgan_loss_grad_huber": lambda: lib.dgan_loss_grad_huber(None, delta, None, None, 1, 1, None, None, None, None,
                                                                 None, 0, None),
        "dgan_loss_grad_measured_huber": lambda: lib.dgan_loss_grad_measured_huber(
            None, delta, None, 10, None, 1, 1, None, None, None, None, None, 0, None),
        "dgan_loss_grad_measured_csr_huber": lambda: lib.dgan_loss_grad_measured_csr_huber(
            None, delta, None, None, None, 10, 5, None, 1, 1, None, None, None, None, None, 0, None)}


@pytest.mark.parametrize("delta", BAD + [1.0, float("inf")])
def test_c_entries_run_the_counterparts_checks_first(delta):
    """Without a handle every entry fails the counterpart's NULL check, whatever delta: delta comes after it."""
    from defensegan_b200 import _native
    lib = _native.load_library()
    for sym, call in _entries(lib, delta).items():
        assert call() == -1, sym
        msg = lib.dgan_last_error().decode()
        assert msg in ("NULL argument", "invalid argument"), (sym, msg)
    bad_adam = ctypes.byref(_native.dgan_adam_params(1.0, 0.999, 1e-8))
    for sym in ("dgan_reconstruct_huber", "dgan_reconstruct_measured_huber", "dgan_reconstruct_measured_csr_huber"):
        assert _entries(lib, delta, bad_adam)[sym]() == -1
        assert "invalid Adam parameters" in lib.dgan_last_error().decode(), sym


@pytest.mark.parametrize("bad", BAD + [True, "0.1", None, [0.1]])
def test_check_huber_delta_names_the_bad_value(bad):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match="huber_delta"):
        _native.check_huber_delta(bad)


def test_check_huber_delta_accepts_positive_values_and_inf_as_fp32():
    from defensegan_b200 import _native
    assert _native.check_huber_delta(float("inf")) == float("inf")
    assert _native.check_huber_delta(2) == 2.0
    assert _native.check_huber_delta(np.float64(0.1)) == float(np.float32(0.1))
    assert _native.check_huber_delta(1e-30) > 0
    # beyond fp32's or even a double's range: +inf as fp32 reads it, or a ValueError naming the value
    assert _native.check_huber_delta(1e40) == float("inf") and _native.check_huber_delta(10 ** 400) == float("inf")
    with pytest.raises(ValueError, match="huber_delta"):
        _native.check_huber_delta(-10 ** 400)


# ---- the binding's routing ----

def test_binding_routes_image_calls_to_the_huber_entries(cpu_native):  # noqa: F811
    x = torch.rand(3, 28, 28, 1)
    pw = torch.ones(3, 28, 28, 1)
    cpu_native.reconstruct(x, 4, 9, 0.5, seed=5, huber_delta=0.25, out=Out(3 * 784))
    cpu_native.reconstruct(x, 4, 9, 0.01, adam=(0.8, 0.99, 1e-6), pixel_weights=pw, prune=[(2, 3)], huber_delta=float("inf"),
                           out=Out(3 * 784))
    cpu_native.loss_grad(x, torch.rand(12, 8), 4, huber_delta=0.5)
    cpu_native.loss_grad(x, torch.rand(12, 8), 4, pixel_weights=pw, huber_delta=0.5)
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes", "dgan_reconstruct_huber", "dgan_workspace_bytes_adam", "dgan_reconstruct_huber",
                     "dgan_workspace_bytes", "dgan_loss_grad_huber", "dgan_workspace_bytes_weighted", "dgan_loss_grad_huber"]
    rc0, rc1 = cpu_native.calls[1][1], cpu_native.calls[3][1]
    assert rc0[2] is None and rc0[3] == 0.25 and rc0[4] is None and rc0[5] == 0 and rc0[7].value is None
    assert rc1[2] is not None and rc1[3] == float("inf") and rc1[5] == 1 and rc1[7].value is not None
    assert cpu_native.calls[2][1][1:4] == (3, 4, 1) and cpu_native.calls[2][1][5] == 1   # the Adam sizer, weighted, P = 1
    lg0, lg1 = cpu_native.calls[5][1], cpu_native.calls[7][1]
    assert lg0[1] == 0.5 and lg0[3].value is None and lg0[4:6] == (3, 4)
    assert lg1[3].value is not None


def test_binding_routes_measured_calls_to_the_huber_entries(cpu_native):  # noqa: F811
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 1.0
    y = torch.rand(3, 10)
    cpu_native.reconstruct_measured(y, a, 4, 9, 1.0, huber_delta=0.1, out=Out(3 * 784))
    cpu_native.reconstruct_measured(y, a.to_sparse_csr(), 4, 9, 0.01, adam=(0.9, 0.999, 1e-8), prune=[(3, 2)],
                                    huber_delta=0.1, out=Out(3 * 784))
    cpu_native.loss_grad_measured(y, a, torch.rand(12, 8), 4, huber_delta=0.1)
    cpu_native.loss_grad_measured(y, a.to_sparse_csr(), torch.rand(12, 8), 4, huber_delta=0.1)
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_measured", "dgan_reconstruct_measured_huber",
                     "dgan_workspace_bytes_measured_adam", "dgan_reconstruct_measured_csr_huber",
                     "dgan_workspace_bytes_measured", "dgan_loss_grad_measured_huber",
                     "dgan_workspace_bytes_measured_csr", "dgan_loss_grad_measured_csr_huber"]
    rc0, rc1 = cpu_native.calls[1][1], cpu_native.calls[3][1]
    assert rc0[2] is None and rc0[3] == pytest.approx(0.1) and rc0[5] == 0 and rc0[7] == 10
    assert rc1[2] is not None and rc1[5] == 1 and rc1[9:11] == (10, 10)
    assert cpu_native.calls[5][1][1] == pytest.approx(0.1) and cpu_native.calls[5][1][3] == 10
    assert cpu_native.calls[7][1][5:7] == (10, 10)


def test_binding_without_huber_routes_exactly_as_before(cpu_native):  # noqa: F811
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    cpu_native.reconstruct(x, 2, 5, out=Out(3 * 784))
    cpu_native.reconstruct(x, 2, 5, huber_delta=None, prune=[(2, 1)], adam=(0.9, 0.999, 1e-8), out=Out(3 * 784))
    cpu_native.loss_grad(x, torch.rand(6, 8), 2, huber_delta=None)
    cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, huber_delta=None, out=Out(3 * 784))
    cpu_native.loss_grad_measured(torch.rand(3, 10), a.to_sparse_csr(), torch.rand(6, 8), 2, huber_delta=None)
    assert [c[0] for c in cpu_native.calls] == [
        "dgan_workspace_bytes", "dgan_reconstruct", "dgan_workspace_bytes_adam", "dgan_reconstruct_adam",
        "dgan_workspace_bytes", "dgan_loss_grad", "dgan_workspace_bytes_measured", "dgan_reconstruct_measured",
        "dgan_workspace_bytes_measured_csr", "dgan_loss_grad_measured_csr"]


def test_binding_refuses_a_bad_delta_before_any_native_call(cpu_native):  # noqa: F811
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    for bad in BAD:
        with pytest.raises(ValueError, match="huber_delta"):
            cpu_native.reconstruct(x, 2, 5, huber_delta=bad)
        with pytest.raises(ValueError, match="huber_delta"):
            cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, huber_delta=bad)
        with pytest.raises(ValueError, match="huber_delta"):
            cpu_native.loss_grad(x, torch.rand(6, 8), 2, huber_delta=bad)
        with pytest.raises(ValueError, match="huber_delta"):
            cpu_native.loss_grad_measured(torch.rand(3, 10), a, torch.rand(6, 8), 2, huber_delta=bad)
    assert cpu_native.calls == []


# ---- DefenseGANBase ----

def test_defaults_and_cfg_key():
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils.config import load_config, packaged_cfg_path
    assert MnistDefenseGAN(test_mode=True, verbose=False).rec_huber_delta is None
    cfg = dict(load_config(packaged_cfg_path("mnist")))
    cfg["REC_HUBER_DELTA"] = 0.1
    assert MnistDefenseGAN(cfg=cfg, test_mode=True, verbose=False).rec_huber_delta == 0.1


def test_squared_error_calls_keep_their_kwargs_and_huber_calls_add_the_delta():
    gan, seen = recording_gan()
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10)] = 1.0
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    assert sorted(seen[0][1]) == ["decay_lr", "momentum", "out", "return_aux", "seed", "z_init_val", "z_row_offset"]
    assert "huber_delta" not in seen[1][1]
    gan.rec_huber_delta = 0.3
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    gan.reconstruct_measured(torch.rand(2, 10), a.to_sparse_csr(), prune=[(10, 2)])
    gan.rec_huber_delta = float("inf")
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    for _, kw in seen[2:5]:
        assert kw["huber_delta"] == pytest.approx(0.3)
    assert seen[4][1]["prune"] == [(10, 2)] and seen[5][1]["huber_delta"] == float("inf")


@pytest.mark.parametrize("val", [0.0, -0.5, float("nan"), "x"])
def test_bad_rec_huber_delta_is_refused_before_any_native_call(val):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    gan.rec_huber_delta = val
    with pytest.raises(ValueError, match="rec_huber_delta"):
        gan.reconstruct(torch.rand(2, 28, 28, 1))
    with pytest.raises(ValueError, match="rec_huber_delta"):
        gan.reconstruct_measured(torch.rand(2, 10), torch.eye(784)[:10])
    with pytest.raises(ValueError, match="rec_huber_delta"):
        gan.rec_cache_dir("test")


def test_rec_cache_dir_names_the_delta_and_parses_back(tmp_path):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils import experiment as E
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 10.0, 200
    plain = gan.rec_cache_dir("test")
    gan.rec_huber_delta = 0.1
    hub = gan.rec_cache_dir("test")
    assert hub.endswith(os.path.join("recs_rr10_lr10.00000_iters200_huber0.1", "test"))
    gan.rec_prune, gan.rec_optimizer, gan.rec_huber_delta = [(40, 2)], "adam", 2.5e-05
    both = gan.rec_cache_dir("dev", max_num=100)
    assert both.endswith(os.path.join("recs_rr10_lr10.00000_iters200_num100_prune40x2_adam0.9-0.999-1e-08_huber2.5e-05",
                                      "dev"))
    gan.rec_huber_delta = float("inf")
    inf = gan.rec_cache_dir("test")
    assert inf.endswith("_huberinf" + os.sep + "test")
    gan.rec_prune, gan.rec_optimizer, gan.rec_huber_delta = None, "momentum", None
    assert gan.rec_cache_dir("test") == plain

    def parsed(path):
        other = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
        other.rec_huber_delta = 7.0                         # overwritten by whatever the name says
        E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=path, override=False,
                                                  online_training=False, train_on_recs=False))
        return other

    assert parsed(plain).rec_huber_delta is None
    assert parsed(hub).rec_huber_delta == pytest.approx(0.1)
    assert parsed(inf).rec_huber_delta == float("inf")
    other = parsed(both)
    assert other.rec_huber_delta == pytest.approx(2.5e-05) and other.rec_optimizer == "adam"
    assert other.rec_cache_dir("dev", max_num=100) == both        # the parsed values name the same directory again


# ---- the oracle ----

def _setup(arch="mnist", b=2, rr=3, seed=0):
    from oracle import defensegan_oracle as O
    weights = O.init_generator_weights(arch, seed=seed, latent_dim=16, net_dim=16, random_bias=True)
    hw, c = (28, 1) if arch == "mnist" else (64, 3)
    rng = np.random.RandomState(seed)
    lo = 0.0 if arch == "mnist" else -1.0
    x = rng.uniform(lo, 1.0, (b, hw, hw, c)).astype(np.float32)
    latent = weights["Generator.Input/Generator.Input.W"].shape[0]
    z0 = O.sample_z0(b * rr, latent, 7)
    return O, weights, x, z0


def test_terms_are_twice_torch_huber_loss_and_clip_follows_the_rules():
    import huber_oracle as H
    d = torch.tensor([-3.0, -0.5, 0.0, 0.2, 1.0, 2.5, float("nan")], dtype=torch.float64)
    w = torch.tensor([1.0, 0.5, 1.0, 0.0, 1.0, 0.25, 1.0], dtype=torch.float64)
    for delta in (0.3, 1.0, 2.0):
        want = 2 * torch.nn.functional.huber_loss(d, torch.zeros_like(d), delta=delta, reduction="none")
        got = H.terms(d, delta)
        assert torch.allclose(got[:-1], want[:-1], rtol=0, atol=1e-15) and torch.isnan(got[-1])
        assert torch.allclose(H.terms(d, delta, w)[:-1], (w * want)[:-1], rtol=0, atol=1e-15)
        c = H.clip(d, delta)
        assert (c[:-1].abs() <= delta).all() and (c[:-1].abs() <= d[:-1].abs()).all() and torch.isnan(c[-1])
    assert torch.equal(H.terms(d[:-1], float("inf")), d[:-1] * d[:-1])


def test_oracle_at_inf_reproduces_the_squared_error_oracles():
    import adam_oracle as AO
    import huber_oracle as H
    import measured_oracle as MO
    import weighted_oracle as WO
    O, weights, x, z0 = _setup()
    inf, rr = float("inf"), 3
    # loss and gradient: the image loss and the measured loss to the bit, the weighted loss's value to the bit
    y0, l0, g0 = O.loss_and_grad("mnist", weights, x, z0, rr, dtype=torch.float64)
    y1, l1, g1 = H.loss_and_grad("mnist", weights, z0, rr, inf, images=x)
    assert np.array_equal(l0, l1) and np.array_equal(g0, g1) and np.array_equal(y0, y1)
    a = MO.gaussian_operator(40, 784, seed=1)
    ym = np.random.RandomState(3).standard_normal((2, 40)).astype(np.float32)
    _, l0, g0 = MO.loss_and_grad("mnist", weights, a, ym, z0, rr, dtype=torch.float64)
    _, l1, g1 = H.loss_and_grad("mnist", weights, z0, rr, inf, operator=a, measurements=ym)
    assert np.array_equal(l0, l1) and np.array_equal(g0, g1)
    pw = np.random.RandomState(4).uniform(0, 1, x.shape).astype(np.float32)
    _, l0, g0 = WO.loss_and_grad("mnist", weights, x, z0, rr, dtype=torch.float64, pixel_weights=pw)
    _, l1, g1 = H.loss_and_grad("mnist", weights, z0, rr, inf, images=x, pixel_weights=pw)
    assert np.array_equal(l0, l1) and np.allclose(g0, g1, rtol=1e-12, atol=1e-15)
    # the R x L loops, momentum and Adam
    r0 = O.reconstruct("mnist", weights, x, rr, 6, rec_lr=10.0, z_init_val=z0, dtype=torch.float64)
    r1 = H.reconstruct("mnist", weights, rr, 6, 10.0, inf, images=x, z_init_val=z0)
    for k in ("loss_all", "rec_all", "idx", "z_final"):
        assert np.array_equal(r0[k], r1[k]), k
    adam = (0.9, 0.999, 1e-8)
    r0 = AO.reconstruct("mnist", weights, rr, 6, 0.05, adam, operator=a, measurements=ym, z_init_val=z0)
    r1 = H.reconstruct("mnist", weights, rr, 6, 0.05, inf, operator=a, measurements=ym, z_init_val=z0, adam=adam)
    for k in ("loss_all", "rec_all", "idx", "z_final"):
        assert np.array_equal(r0[k], r1[k]), k
    r0 = AO.reconstruct("mnist", weights, rr, 6, 0.05, adam, images=x, pixel_weights=pw, z_init_val=z0)
    r1 = H.reconstruct("mnist", weights, rr, 6, 0.05, inf, images=x, pixel_weights=pw, z_init_val=z0, adam=adam)
    for k in ("loss_all", "rec_all", "z_final"):
        assert np.allclose(r0[k], r1[k], rtol=1e-10, atol=1e-12), k


@pytest.mark.parametrize("case", ["image", "weighted", "measured"])
def test_oracle_gradient_matches_finite_differences(case):
    import huber_oracle as H
    import measured_oracle as MO
    O, weights, x, z0 = _setup()
    rr, delta = 3, 0.1
    kw = dict(images=x)
    if case == "weighted":
        kw["pixel_weights"] = np.random.RandomState(4).uniform(0, 1, x.shape).astype(np.float32)
    if case == "measured":
        a = MO.gaussian_operator(40, 784, seed=1)
        kw = dict(operator=a, measurements=np.random.RandomState(3).standard_normal((2, 40)).astype(np.float32) * 0.3)
    _, loss, g = H.loss_and_grad("mnist", weights, z0, rr, delta, **kw)
    # a Huber loss with clipping: some residuals beyond delta, some within
    y, _, _ = H.loss_and_grad("mnist", weights, z0, rr, float("inf"), **kw)
    rng = np.random.RandomState(5)
    z = z0.astype(np.float64)
    for _ in range(3):
        v = rng.standard_normal(z.shape)
        v /= np.linalg.norm(v)
        h = 1e-6
        lp = H.loss_and_grad("mnist", weights, z + h * v, rr, delta, **kw)[1].sum()
        lm = H.loss_and_grad("mnist", weights, z - h * v, rr, delta, **kw)[1].sum()
        fd = (lp - lm) / (2 * h)
        assert fd == pytest.approx(float((g * v).sum()), rel=1e-5, abs=1e-9)
    assert math.isfinite(float(loss.sum()))
