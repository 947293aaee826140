"""CPU tests (no GPU) of restart pruning (dgan_reconstruct_pruned): the schedule checks of the binding and of
DefenseGANBase (raised before any native call), the use_bn and reconstruct_measured refusals, and the cache-directory naming
and its parse-back."""
import ctypes
import os

import pytest
import torch

from recording import Out, cpu_native  # noqa: F401  (the fixture)


def test_sizer_and_layout_refuse_bad_schedules_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(40, 2))
    assert lib.dgan_workspace_bytes_pruned(None, 4, 10, sched, 1, 0) == 0
    assert lib.dgan_workspace_bytes_pruned(None, 4, 10, None, 0, 0) == 0
    fn = lib.dgan_debug_workspace_layout_pruned
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_native.dgan_prune_point), ctypes.c_int,
                   ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    buf = ctypes.create_string_buffer(1 << 12)
    assert fn(None, 4, 10, sched, 1, 0, buf, len(buf)) == -1


# ---- the schedule rules ----

GOOD = [([(40, 2)], 10, 200), ([(20, 5), (60, 2), (120, 1)], 10, 200), ([(1, 10)], 10, 2), ([(199, 1)], 10, 200),
        ([(5, 3), (6, 3)], 3, 7)]
BAD = [([], 10, 200, "at least one"),
       ([(0, 2)], 10, 200, r"point 0 \(iter 0, keep 2\): iter must be >= 1"),
       ([(200, 2)], 10, 200, r"point 0 .*<= rec_iters - 1 = 199"),
       ([(40, 11)], 10, 200, r"point 0 .*keep must be <= rec_rr = 10"),
       ([(40, 0)], 10, 200, r"point 0 .*keep must be >= 1"),
       ([(40, 2), (40, 1)], 10, 200, r"point 1 \(iter 40, keep 1\): iter must exceed"),
       ([(40, 2), (30, 1)], 10, 200, r"point 1 .*iter must exceed"),
       ([(40, 2), (60, 3)], 10, 200, r"point 1 \(iter 60, keep 3\): keep must not exceed"),
       ([(40, 2.0)], 10, 200, r"point 0 .*pair of integers"),
       ([(40,)], 10, 200, r"point 0 .*pair of integers"),
       ([40, 2], 10, 200, r"sequence of \(iter, keep\) pairs|point 0"),
       ([(True, 2)], 10, 200, r"point 0 .*pair of integers")]


@pytest.mark.parametrize("sched,rr,iters", GOOD)
def test_check_prune_schedule_accepts(sched, rr, iters):
    from defensegan_b200 import _native
    assert _native.check_prune_schedule([list(p) for p in sched], rr, iters) == sched


@pytest.mark.parametrize("sched,rr,iters,match", BAD)
def test_check_prune_schedule_names_the_bad_point(sched, rr, iters, match):
    from defensegan_b200 import _native
    with pytest.raises(ValueError, match=match):
        _native.check_prune_schedule(sched, rr, iters)


# ---- the binding: the schedule reaches the pruned entry unchanged ----

@pytest.mark.parametrize("weighted", [False, True])
def test_binding_passes_the_schedule_to_the_pruned_entry(cpu_native, weighted):
    x = torch.rand(3, 28, 28, 1)
    pw = torch.ones_like(x) if weighted else None
    cpu_native.reconstruct(x, 4, 9, 2.5, seed=5, pixel_weights=pw, prune=[(2, 3), (5, 1)], out=cpu_native.Out(x.numel()))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_pruned", "dgan_reconstruct_pruned"]
    _, (_, b, rr, sched, n, w) = cpu_native.calls[0]
    assert (b, rr, n, w) == (3, 4, 2, int(weighted))
    assert [(sched[i].iter, sched[i].keep) for i in range(n)] == [(2, 3), (5, 1)]
    args = cpu_native.calls[1][1]
    assert args[2] is sched and args[3] == 2
    assert (args[5].value is not None) == weighted          # w_dev: NULL unweighted


def test_binding_without_a_schedule_runs_the_plain_entries(cpu_native):
    x = torch.rand(2, 28, 28, 1)
    cpu_native.reconstruct(x, 2, 5, out=cpu_native.Out(x.numel()))
    cpu_native.reconstruct(x, 2, 5, pixel_weights=torch.ones_like(x), out=cpu_native.Out(x.numel()))
    assert [c[0] for c in cpu_native.calls] == ["dgan_workspace_bytes", "dgan_reconstruct",
                                                "dgan_workspace_bytes_weighted", "dgan_reconstruct_weighted"]


def test_binding_refuses_bad_schedules_and_use_bn_before_any_native_call(cpu_native):
    x = torch.rand(2, 28, 28, 1)
    with pytest.raises(ValueError, match="point 0"):
        cpu_native.reconstruct(x, 2, 5, prune=[(5, 1)])
    cpu_native.use_bn = True
    with pytest.raises(ValueError, match="use_bn"):
        cpu_native.reconstruct(x, 2, 5, prune=[(2, 1)])
    assert cpu_native.calls == []


# ---- DefenseGANBase ----

def _gan(**kw):
    """A model whose native calls fail loudly: the checks under test must come first."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, **kw)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    return gan


def test_rec_prune_defaults_to_none_and_is_set_from_the_cfg():
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils.config import packaged_cfg_path, load_config
    assert MnistDefenseGAN(test_mode=True, verbose=False).rec_prune is None
    cfg = load_config(packaged_cfg_path("mnist"))
    cfg["REC_PRUNE"] = [[40, 2], [120, 1]]
    assert MnistDefenseGAN(cfg=cfg, test_mode=True, verbose=False).rec_prune == [[40, 2], [120, 1]]


@pytest.mark.parametrize("sched,match", [([(0, 2)], "point 0"), ([(40, 2), (30, 1)], "point 1"), ([(40, 11)], "rec_rr"),
                                         ([(200, 1)], "rec_iters - 1")])
def test_reconstruct_checks_the_schedule_before_any_native_call(sched, match):
    gan = _gan()
    gan.rec_rr, gan.rec_iters, gan.rec_prune = 10, 200, sched
    with pytest.raises(ValueError, match=match):
        gan.reconstruct(torch.rand(2, 28, 28, 1))


def test_reconstruct_refuses_pruning_with_use_bn_before_any_native_call():
    gan = _gan(use_bn=True)
    gan.rec_prune = [(40, 2)]
    with pytest.raises(ValueError, match="use_bn"):
        gan.reconstruct(torch.rand(2, 28, 28, 1))


def test_reconstruct_measured_refuses_pruning_before_any_native_call():
    gan = _gan()
    gan.rec_prune = [(40, 2)]
    with pytest.raises(ValueError, match="rec_prune"):
        gan.reconstruct_measured(torch.rand(2, 10), torch.rand(10, 784))


def test_defensegan_passes_the_checked_schedule():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    seen = {}

    class FakeNative:
        def reconstruct(self, x, *args, **kw):
            seen.update(kw)
            return x

    gan._as_cuda = lambda t: t.to(torch.float32)
    gan._get_native = lambda device: FakeNative()
    gan.rec_rr, gan.rec_iters = 4, 50
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    assert "prune" not in seen                                  # unset: today's call
    gan.rec_prune = [[10, 2], [20, 1]]                          # as a YAML list of pairs arrives
    gan.reconstruct(torch.rand(2, 28, 28, 1))
    assert seen["prune"] == [(10, 2), (20, 1)]


# ---- the cache directory ----

def test_rec_cache_dir_names_the_schedule_and_parses_back(tmp_path):
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200.utils import experiment as E
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 10.0, 200
    plain = gan.rec_cache_dir("test")
    plain_num = gan.rec_cache_dir("dev", max_num=100)
    assert plain.endswith(os.path.join("recs_rr10_lr10.00000_iters200", "test"))
    gan.rec_prune = [(20, 5), (60, 2), (120, 1)]
    pruned = gan.rec_cache_dir("test")
    assert pruned.endswith(os.path.join("recs_rr10_lr10.00000_iters200_prune20x5-60x2-120x1", "test"))
    assert gan.rec_cache_dir("dev", max_num=100).endswith(
        os.path.join("recs_rr10_lr10.00000_iters200_num100_prune20x5-60x2-120x1", "dev"))
    gan.rec_prune = [(40, 2)]
    one = gan.rec_cache_dir("train")
    assert one.endswith(os.path.join("recs_rr10_lr10.00000_iters200_prune40x2", "train"))
    gan.rec_prune = None
    assert gan.rec_cache_dir("test") == plain and gan.rec_cache_dir("dev", max_num=100) == plain_num

    def parse(path):
        other = MnistDefenseGAN(test_mode=True, verbose=False)
        other.rec_prune = [(1, 1)]                              # overwritten by whatever the name says
        E.set_test_time_rec_params(other, E.Flags(defense_type="defense_gan", rec_path=path, override=False,
                                                  online_training=False, train_on_recs=False))
        return other.rec_rr, other.rec_lr, other.rec_iters, other.rec_prune

    assert parse(pruned) == (10, 10.0, 200, [(20, 5), (60, 2), (120, 1)])
    assert parse(one) == (10, 10.0, 200, [(40, 2)])
    assert parse(plain) == (10, 10.0, 200, None)
    assert parse(plain_num) == (10, 10.0, 200, None)
