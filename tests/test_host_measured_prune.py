"""CPU tests (no GPU) of restart pruning in the projection from linear measurements (dgan_reconstruct_measured_pruned,
dgan_reconstruct_measured_csr_pruned): the binding's routing of dense, COO and CSR operators with and without a
schedule, the three `prune` cases of DefenseGANBase.reconstruct_measured with their refusals raised before any native
call.  The layout of a pruned measured workspace needs a handle, so tests/test_gpu_measured_prune.py reads it; here the
printer's refusal without one."""
import ctypes
import os

import pytest
import torch

from recording import Out, cpu_native  # noqa: F401  (the fixture)


def _layout_fn(lib):
    from defensegan_b200 import _native
    fn = lib.dgan_debug_workspace_layout_measured_pruned
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                   ctypes.POINTER(_native.dgan_prune_point), ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    return fn


def test_sizer_and_layout_refuse_bad_arguments_without_a_handle():
    from defensegan_b200 import _native
    lib = _native.load_library()
    sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(40, 2))
    assert lib.dgan_workspace_bytes_measured_pruned(None, 4, 10, 100, -1, sched, 1) == 0
    assert lib.dgan_workspace_bytes_measured_pruned(None, 4, 10, 100, 50, None, 0) == 0
    buf = ctypes.create_string_buffer(1 << 12)
    assert _layout_fn(lib)(None, 4, 10, 100, -1, sched, 1, buf, len(buf)) == -1


# ---- the binding's routing ----

def _operators():
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 1.0
    return a, a.to_sparse_csr()


def test_binding_routes_dense_and_csr_with_a_schedule_to_the_pruned_entries(cpu_native):
    a, acsr = _operators()
    y = torch.rand(3, 10)
    cpu_native.reconstruct_measured(y, a, 4, 9, 2.5, seed=5, prune=[(2, 3), (5, 1)], out=Out(3 * 784))
    cpu_native.reconstruct_measured(y, acsr, 4, 9, 2.5, seed=5, prune=[[2, 3], [5, 1]], out=Out(3 * 784))
    names = [c[0] for c in cpu_native.calls]
    assert names == ["dgan_workspace_bytes_measured_pruned", "dgan_reconstruct_measured_pruned",
                     "dgan_workspace_bytes_measured_pruned", "dgan_reconstruct_measured_csr_pruned"]
    for k, nnz in ((0, -1), (2, 10)):
        _, (_, b, rr, m, nz, sched, n) = cpu_native.calls[k]
        assert (b, rr, m, nz, n) == (3, 4, 10, nnz, 2)
        assert [(sched[i].iter, sched[i].keep) for i in range(n)] == [(2, 3), (5, 1)]
        args = cpu_native.calls[k + 1][1]
        assert args[2] is sched and args[3] == 2
    dense_args, csr_args = cpu_native.calls[1][1], cpu_native.calls[3][1]
    assert dense_args[5] == 10                                 # a_dev, m
    assert csr_args[7:9] == (10, 10)                           # row_ptr, col_idx, val, m, nnz


def test_binding_without_a_schedule_routes_exactly_as_before(cpu_native):
    a, acsr = _operators()
    y = torch.rand(3, 10)
    cpu_native.reconstruct_measured(y, a, 2, 5, out=Out(3 * 784))
    cpu_native.reconstruct_measured(y, acsr, 2, 5, prune=None, out=Out(3 * 784))
    assert [c[0] for c in cpu_native.calls] == ["dgan_workspace_bytes_measured", "dgan_reconstruct_measured",
                                                "dgan_workspace_bytes_measured_csr", "dgan_reconstruct_measured_csr"]
    assert cpu_native.calls[0][1][1:] == (3, 2, 10)
    assert cpu_native.calls[2][1][1:] == (3, 2, 10, 10)


def test_binding_refuses_bad_schedules_and_use_bn_before_any_native_call(cpu_native):
    a, acsr = _operators()
    y = torch.rand(3, 10)
    for op in (a, acsr):
        with pytest.raises(ValueError, match="point 0"):
            cpu_native.reconstruct_measured(y, op, 2, 5, prune=[(5, 1)])
        with pytest.raises(ValueError, match="point 1"):
            cpu_native.reconstruct_measured(y, op, 4, 9, prune=[(2, 2), (3, 3)])
    cpu_native.use_bn = True
    with pytest.raises(ValueError, match="use_bn"):
        cpu_native.reconstruct_measured(y, a, 2, 5, prune=[(2, 1)])
    assert cpu_native.calls == []


# ---- DefenseGANBase.reconstruct_measured ----

def _gan(**kw):
    """A model whose native calls fail loudly: the checks under test must come first."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, **kw)

    def no_native(*a, **k):
        raise AssertionError("a native call was made")

    gan._get_native = no_native
    gan._as_cuda = no_native
    return gan


def _recording_gan():
    """A model whose native generator records the prune argument of each reconstruct_measured call."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    seen = []

    class FakeNative:
        def reconstruct_measured(self, y, a, *args, **kw):
            seen.append((a.layout, kw["prune"]))
            return y

    gan._as_cuda = lambda t: t.to(torch.float32)
    gan._get_native = lambda device: FakeNative()
    gan.rec_rr, gan.rec_iters = 4, 50
    return gan, seen


def _three_operators():
    a = torch.zeros(10, 784)
    a[torch.arange(10), torch.arange(10) * 7] = 0.5
    return [a, a.to_sparse(), a.to_sparse_csr()]


def test_prune_not_given_is_todays_call():
    gan, seen = _recording_gan()
    y = torch.rand(2, 10)
    for op in _three_operators():
        gan.reconstruct_measured(y, op)
    assert [p for _, p in seen] == [None, None, None]
    assert [lay for lay, _ in seen] == [torch.strided, torch.sparse_csr, torch.sparse_csr]


def test_prune_not_given_with_rec_prune_set_is_refused_before_any_native_call():
    gan = _gan()
    gan.rec_prune = [(40, 2)]
    for op in _three_operators():
        with pytest.raises(ValueError, match="rec_prune"):
            gan.reconstruct_measured(torch.rand(2, 10), op)


def test_prune_given_reaches_the_native_call_checked():
    gan, seen = _recording_gan()
    gan.rec_prune = [(7, 1)]                                    # ignored: the call names its own schedule
    y = torch.rand(2, 10)
    for op in _three_operators():
        gan.reconstruct_measured(y, op, prune=[[10, 2], [20, 1]])
    assert [p for _, p in seen] == [[(10, 2), (20, 1)]] * 3


def test_prune_none_given_is_an_unpruned_call_whatever_rec_prune_holds():
    gan, seen = _recording_gan()
    gan.rec_prune = [(10, 2)]
    y = torch.rand(2, 10)
    for op in _three_operators():
        gan.reconstruct_measured(y, op, prune=None)
    assert [p for _, p in seen] == [None, None, None]


@pytest.mark.parametrize("sched,match", [([(0, 2)], "point 0"), ([(40, 2), (30, 1)], "point 1"), ([(40, 11)], "rec_rr"),
                                         ([(200, 1)], "rec_iters - 1"), ([], "at least one")])
def test_prune_is_checked_before_any_native_call(sched, match):
    gan = _gan()
    gan.rec_rr, gan.rec_iters = 10, 200
    for op in _three_operators():
        with pytest.raises(ValueError, match=match):
            gan.reconstruct_measured(torch.rand(2, 10), op, prune=sched)


def test_prune_is_refused_with_use_bn_before_any_native_call():
    gan = _gan(use_bn=True)
    gan.rec_rr, gan.rec_iters = 10, 200
    for op in _three_operators():
        with pytest.raises(ValueError, match="use_bn"):
            gan.reconstruct_measured(torch.rand(2, 10), op, prune=[(40, 2)])
    with pytest.raises(AssertionError, match="native call"):          # prune=None with use_bn: not refused here
        gan.reconstruct_measured(torch.rand(2, 10), _three_operators()[0], prune=None)
