"""CPU tests (no GPU) of the Adam update of the latent rows (dgan_reconstruct_adam, dgan_reconstruct_measured_adam,
dgan_reconstruct_measured_csr_adam): the refusal of bad Adam parameters by the C entries and by Python before any native
call, the binding's routing (and a momentum call's kwargs unchanged), DefenseGANBase's rec_optimizer attributes, and the
cache name and its parse-back.  The Adam workspace's layout needs a handle, so tests/test_gpu_adam.py reads it."""
import ctypes
import os

import pytest
import torch

from recording import Out, cpu_native, recording_gan  # noqa: F401  (the fixture)

BAD = [((1.0, 0.999, 1e-8), "beta1"), ((-0.5, 0.999, 1e-8), "beta1"), ((float("nan"), 0.999, 1e-8), "beta1"),
       ((0.9, 1.0, 1e-8), "beta2"), ((0.9, -1e-3, 1e-8), "beta2"), ((0.9, 0.999, 0.0), "eps"),
       ((0.9, 0.999, -1e-8), "eps"), ((0.9, 0.999, float("inf")), "eps"), ((0.9, 0.999, float("nan")), "eps")]


# ---- refusals ----

def _entries(lib, ap):
    """Each Adam entry called with the Adam parameters ap and everything else NULL or 0."""
    return {"dgan_reconstruct_adam": lambda: lib.dgan_reconstruct_adam(None, None, ap, None, 0, None, None, None, None,
                                                                       None, None, None, 0, None),
            "dgan_reconstruct_measured_adam": lambda: lib.dgan_reconstruct_measured_adam(None, None, ap, None, 0, None, 10,
                                                                                         None, None, None, None, None,
                                                                                         None, 0, None),
            "dgan_reconstruct_measured_csr_adam": lambda: lib.dgan_reconstruct_measured_csr_adam(
                None, None, ap, None, 0, None, None, None, 10, 5, None, None, None, None, None, None, 0, None)}


@pytest.mark.parametrize("bad,name", BAD)
def test_c_entries_refuse_bad_adam_parameters_first(bad, name):
    from defensegan_b200 import _native
    lib = _native.load_library()
    ap = ctypes.byref(_native.dgan_adam_params(*bad))
    for sym, call in _entries(lib, ap).items():
        assert call() == -1, sym
        msg = lib.dgan_last_error().decode()
        assert "invalid Adam parameters" in msg and name in msg, (sym, msg)
    for sym, call in _entries(lib, None).items():
        assert call() == -1 and "NULL Adam parameters" in lib.dgan_last_error().decode(), sym
    good = ctypes.byref(_native.dgan_adam_params(0.9, 0.999, 1e-8))
    for sym, call in _entries(lib, good).items():          # good parameters: refused for the NULL handle instead
        assert call() == -1 and lib.dgan_last_error().decode() == "NULL argument", sym


def test_sizers_and_layout_refuse_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(40, 2))
    assert lib.dgan_workspace_bytes_adam(None, 4, 10, 0, None, 0) == 0
    assert lib.dgan_workspace_bytes_adam(None, 4, 10, 1, sched, 1) == 0
    assert lib.dgan_workspace_bytes_measured_adam(None, 4, 10, 100, -1, None, 0) == 0
    fn = lib.dgan_debug_workspace_layout_adam
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                   ctypes.POINTER(_native.dgan_prune_point), ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    buf = ctypes.create_string_buffer(1 << 12)
    assert fn(None, 4, 10, 0, 0, -1, None, 0, buf, len(buf)) == -1


@pytest.mark.parametrize("bad,name", BAD + [((0.9, 0.999), "triple"), ((0.9, "x", 1e-8), "beta2"),
                                            ((0.9, 0.999, True), "eps"), (0.9, "triple")])
def test_check_adam_params_names_the_bad_value(bad, name):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match=name):
        _native.check_adam_params(bad)


def test_check_adam_params_accepts_the_edges_as_fp32():
    from defensegan_b200 import _native
    assert _native.check_adam_params((0, 0.0, 1e-30)) == (0.0, 0.0, float(torch.tensor(1e-30).item()))
    assert _native.check_adam_params([0.9, 0.999, 1e-8])[0] == pytest.approx(0.9)
    with pytest.raises(ValueError, match="beta1"):            # rounds to 1.0 in fp32
        _native.check_adam_params((1 - 1e-9, 0.999, 1e-8))


# ---- the binding's routing ----

def _adam_of(byref):
    p = byref._obj
    return tuple(round(float(getattr(p, f)), 6) for f in ("beta1", "beta2", "eps"))


def test_binding_routes_image_calls_to_the_adam_entry(cpu_native):
    x = torch.rand(3, 28, 28, 1)
    pw = torch.ones(3, 28, 28, 1)
    cpu_native.reconstruct(x, 4, 9, 0.01, seed=5, adam=(0.8, 0.99, 1e-6), out=Out(3 * 784))
    cpu_native.reconstruct(x, 4, 9, 0.01, seed=5, adam=(0.8, 0.99, 1e-6), pixel_weights=pw, prune=[(2, 3), (5, 1)],
                           out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_adam", "dgan_reconstruct_adam"] * 2
    (_, sz0), (_, rc0), (_, sz1), (_, rc1) = cpu_native.calls
    assert sz0[1:] == (3, 4, 0, None, 0)
    assert sz1[1:3] == (3, 4) and sz1[3] == 1 and sz1[5] == 2
    assert [(sz1[4][i].iter, sz1[4][i].keep) for i in range(2)] == [(2, 3), (5, 1)]
    for args, n_points, weighted in ((rc0, 0, False), (rc1, 2, True)):
        assert _adam_of(args[2]) == (0.8, 0.99, 1e-6)
        assert args[4] == n_points and (args[3] is None) == (n_points == 0)
        assert (args[6].value is not None) == weighted              # w_dev NULL without weights


def test_binding_routes_measured_calls_to_the_adam_entries(cpu_native):
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 1.0
    y = torch.rand(3, 10)
    cpu_native.reconstruct_measured(y, a, 4, 9, 0.01, adam=(0.9, 0.999, 1e-8), out=Out(3 * 784))
    cpu_native.reconstruct_measured(y, a.to_sparse_csr(), 4, 9, 0.01, adam=(0.9, 0.999, 1e-8), prune=[(3, 2)],
                                    out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_measured_adam", "dgan_reconstruct_measured_adam",
                     "dgan_workspace_bytes_measured_adam", "dgan_reconstruct_measured_csr_adam"]
    assert cpu_native.calls[0][1][1:] == (3, 4, 10, -1, None, 0)
    assert cpu_native.calls[2][1][1:5] == (3, 4, 10, 10) and cpu_native.calls[2][1][6] == 1
    assert cpu_native.calls[1][1][4] == 0 and cpu_native.calls[1][1][6] == 10          # n_points, m
    assert cpu_native.calls[3][1][4] == 1 and cpu_native.calls[3][1][8:10] == (10, 10)  # n_points, m, nnz


def test_binding_without_adam_routes_exactly_as_before(cpu_native):
    x = torch.rand(3, 28, 28, 1)
    cpu_native.reconstruct(x, 2, 5, out=Out(3 * 784))
    cpu_native.reconstruct(x, 2, 5, adam=None, prune=[(2, 1)], out=Out(3 * 784))
    assert [c[0] for c in cpu_native.calls] == ["dgan_workspace_bytes", "dgan_reconstruct", "dgan_workspace_bytes_pruned",
                                                "dgan_reconstruct_pruned"]


def test_binding_refuses_bad_adam_before_any_native_call(cpu_native):
    x = torch.rand(3, 28, 28, 1)
    a = torch.eye(784)[:10]
    for bad, name in BAD:
        with pytest.raises(ValueError, match=name):
            cpu_native.reconstruct(x, 2, 5, adam=bad)
        with pytest.raises(ValueError, match=name):
            cpu_native.reconstruct_measured(torch.rand(3, 10), a, 2, 5, adam=bad)
    assert cpu_native.calls == []


# ---- DefenseGANBase ----

def test_defaults_and_cfg_keys():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    assert (gan.rec_optimizer, tuple(gan.rec_adam_betas), gan.rec_adam_eps) == ("momentum", (0.9, 0.999), 1e-8)
    from defensegan_b200.utils.config import load_config, packaged_cfg_path
    cfg = dict(load_config(packaged_cfg_path("mnist")))
    cfg.update({"REC_OPTIMIZER": "adam", "REC_ADAM_BETAS": [0.5, 0.9], "REC_ADAM_EPS": 1e-6})
    gan = MnistDefenseGAN(cfg=cfg, test_mode=True, verbose=False)
    assert (gan.rec_optimizer, list(gan.rec_adam_betas), gan.rec_adam_eps) == ("adam", [0.5, 0.9], 1e-6)


def test_momentum_calls_keep_their_kwargs_and_adam_calls_add_adam():
    gan, seen = recording_gan()
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10)] = 1.0
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    assert sorted(seen[0][1]) == ["decay_lr", "momentum", "out", "return_aux", "seed", "z_init_val", "z_row_offset"]
    assert "adam" not in seen[1][1]
    gan.rec_optimizer, gan.rec_adam_betas, gan.rec_adam_eps = "adam", [0.8, 0.99], 1e-6
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    gan.reconstruct_measured(torch.rand(2, 10), a)
    gan.reconstruct_measured(torch.rand(2, 10), a.to_sparse_csr(), prune=[(10, 2)])
    for _, kw in seen[2:]:
        assert kw["adam"] == pytest.approx((0.8, 0.99, 1e-6))
    assert seen[4][1]["prune"] == [(10, 2)]


@pytest.mark.parametrize("attr,val,match", [("rec_optimizer", "sgd", "rec_optimizer"), ("rec_optimizer", "Adam", "rec_optimizer"),
                                            ("rec_adam_betas", (1.0, 0.999), "beta1"),
                                            ("rec_adam_betas", (0.9, 1.5), "beta2"), ("rec_adam_betas", 0.9, "pair"),
                                            ("rec_adam_betas", (0.9,), "pair"), ("rec_adam_eps", 0.0, "eps"),
                                            ("rec_adam_eps", float("nan"), "eps")])
def test_bad_values_are_refused_before_any_native_call(attr, val, match):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    gan.rec_optimizer = "adam"
    setattr(gan, attr, val)
    with pytest.raises(ValueError, match=match):
        gan.reconstruct(torch.rand(2, 28, 28, 1))
    with pytest.raises(ValueError, match=match):
        gan.reconstruct_measured(torch.rand(2, 10), torch.eye(784)[:10])
    with pytest.raises(ValueError, match=match):
        gan.rec_cache_dir("test")


def test_rec_cache_dir_names_adam_and_parses_back(tmp_path):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils import experiment as E
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 0.01, 200
    plain = gan.rec_cache_dir("test")
    assert plain.endswith(os.path.join("recs_rr10_lr0.01000_iters200", "test"))
    gan.rec_optimizer = "adam"
    adam = gan.rec_cache_dir("test")
    assert adam.endswith(os.path.join("recs_rr10_lr0.01000_iters200_adam0.9-0.999-1e-08", "test"))
    gan.rec_prune, gan.rec_adam_betas, gan.rec_adam_eps = [(40, 2)], (0.5, 0.99), 1e-6
    both = gan.rec_cache_dir("dev", max_num=100)
    assert both.endswith(os.path.join("recs_rr10_lr0.01000_iters200_num100_prune40x2_adam0.5-0.99-1e-06", "dev"))
    gan.rec_optimizer, gan.rec_prune = "momentum", None
    assert gan.rec_cache_dir("test") == plain

    def parse(path):
        other = MnistDefenseGAN(test_mode=True, verbose=False)
        other.rec_optimizer = "adam"                            # overwritten by whatever the name says
        E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=path, override=False,
                                                  online_training=False, train_on_recs=False))
        return (other.rec_rr, other.rec_lr, other.rec_iters, other.rec_prune, other.rec_optimizer,
                tuple(other.rec_adam_betas), other.rec_adam_eps)

    assert parse(adam) == (10, 0.01, 200, None, "adam", (0.9, 0.999), 1e-8)
    assert parse(both) == (10, 0.01, 200, [(40, 2)], "adam", (0.5, 0.99), 1e-6)
    assert parse(plain)[4] == "momentum"
    # the parsed values name the same directory again
    other = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=both, override=False,
                                              online_training=False, train_on_recs=False))
    assert other.rec_cache_dir("dev", max_num=100) == both
