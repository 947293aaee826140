"""CPU tests (no GPU) of the Adam update of the latent rows (dgan_reconstruct_adam, dgan_reconstruct_measured_adam,
dgan_reconstruct_measured_csr_adam): the exported symbols against the header, dgan_adam_params against the C compiler,
the refusal of bad Adam parameters by the C entries and by Python before any native call, the binding's routing (and a
momentum call's kwargs unchanged), DefenseGANBase's rec_optimizer attributes, the cache name and its parse-back, and
what ptxas made of the new kernels.  The Adam workspace's layout needs a handle, so tests/test_gpu_adam.py reads it."""
import contextlib
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["dgan_workspace_bytes_adam", "dgan_workspace_bytes_measured_adam", "dgan_reconstruct_adam",
               "dgan_reconstruct_measured_adam", "dgan_reconstruct_measured_csr_adam"]
BAD = [((1.0, 0.999, 1e-8), "beta1"), ((-0.5, 0.999, 1e-8), "beta1"), ((float("nan"), 0.999, 1e-8), "beta1"),
       ((0.9, 1.0, 1e-8), "beta2"), ((0.9, -1e-3, 1e-8), "beta2"), ((0.9, 0.999, 0.0), "eps"),
       ((0.9, 0.999, -1e-8), "eps"), ((0.9, 0.999, float("inf")), "eps"), ((0.9, 0.999, float("nan")), "eps")]


def test_symbols_are_exported_with_the_header_signatures():
    from defensegan_b200 import _native
    lib = _native.load_library()
    header = open(os.path.join(ROOT, "include", "defensegan_b200.h")).read()
    ctype = {"int": ctypes.c_int, "size_t": ctypes.c_size_t}
    for sym in NEW_SYMBOLS:
        assert sym in _native.ABI_SYMBOLS and hasattr(lib, sym)
        m = re.search(r"(\w+)\s+%s\s*\(([^)]*)\)" % sym, header)
        assert m, sym
        want = []
        for p in (" ".join(p.split()) for p in m.group(2).split(",")):
            if "dgan_rec_params" in p:
                want.append(ctypes.POINTER(_native.dgan_rec_params))
            elif "dgan_prune_point" in p:
                want.append(ctypes.POINTER(_native.dgan_prune_point))
            elif "dgan_adam_params" in p:
                want.append(ctypes.POINTER(_native.dgan_adam_params))
            elif "*" in p or p.startswith("dgan_handle"):
                want.append(ctypes.c_void_p)
            else:
                want.append(ctype[p.rsplit(" ", 1)[0]])
        fn = getattr(lib, sym)
        assert list(fn.argtypes) == want, sym
        assert fn.restype == ctype[m.group(1)], sym
    assert lib.dgan_abi_version() == 2


def test_adam_params_struct_matches_the_compilers_layout_and_the_header_is_c99(tmp_path):
    from defensegan_b200 import _native
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "defensegan_b200.h"\n'
                   'int (*f)(dgan_handle, const dgan_rec_params*, const dgan_adam_params*, const dgan_prune_point*, int, '
                   'const int32_t*, const int32_t*, const float*, int, int, const float*, const float*, float*, float*, '
                   'int32_t*, void*, size_t, void*) = dgan_reconstruct_measured_csr_adam;\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(dgan_adam_params), '
                   'offsetof(dgan_adam_params, beta1), offsetof(dgan_adam_params, beta2), offsetof(dgan_adam_params, eps));'
                   ' return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                    "-L", os.path.dirname(_native.LIB_PATH), "-Wl,--unresolved-symbols=ignore-all"], check=True)
    got = tuple(int(v) for v in subprocess.run([str(exe)], stdout=subprocess.PIPE, text=True, check=True).stdout.split())
    A = _native.dgan_adam_params
    assert got == (ctypes.sizeof(A), A.beta1.offset, A.beta2.offset, A.eps.offset)


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

@pytest.fixture
def cpu_native(monkeypatch):
    """A NativeGenerator whose library records its calls (no GPU)."""
    from defensegan_b200 import _native
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            def f(*args):
                calls.append((name, args))
                return 1 << 20 if name.startswith("dgan_workspace_bytes") else 0
            return f

    class Stream:
        cuda_stream = 0

    monkeypatch.setattr(_native, "_require_cuda_f32", lambda t, name: t.to(torch.float32).contiguous())
    monkeypatch.setattr(_native, "_require_cuda_i32", lambda t, name: t.to(torch.int32).contiguous())
    monkeypatch.setattr(_native, "_require_aligned_out", lambda rec: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: Stream())
    g = object.__new__(_native.NativeGenerator)
    g.lib, g.device, g._ws, g._handle = FakeLib(), torch.device("cpu"), None, ctypes.c_void_p(0)
    g.image_dim, g.hwc, g.latent_dim, g.use_bn = (28, 28, 1), 784, 8, False
    g.calls = calls
    return g


class Out:
    """Stands in for a CUDA `out` tensor of n elements."""
    is_cuda, dtype = True, torch.float32

    def __init__(self, n):
        self.n = n

    def is_contiguous(self):
        return True

    def numel(self):
        return self.n

    def data_ptr(self):
        return 0


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

def _recording_gan(**kw):
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, **kw)
    seen = []

    class FakeNative:
        def reconstruct(self, x, *args, **kw):
            seen.append(("reconstruct", kw))
            return x

        def reconstruct_measured(self, y, a, *args, **kw):
            seen.append(("reconstruct_measured", kw))
            return y

    gan._as_cuda = lambda t: t.to(torch.float32)
    gan._get_native = lambda device: FakeNative()
    gan.rec_rr, gan.rec_iters = 4, 50
    return gan, seen


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
    gan, seen = _recording_gan()
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


# ---- what ptxas made of the new kernels ----

def test_adam_kernels_compile_for_sm90a_without_spills(tmp_path):
    from defensegan_b200 import _native
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = tmp_path / "adam.cu"
    src.write_text('#include "%s"\n' % os.path.join(_native.CSRC_DIR, "kernels_adam.cuh"))
    flags = [f for f in _native.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    res = subprocess.run([nvcc] + flags + ["-cubin", "-Xptxas", "-v", str(src), "-o", str(tmp_path / "adam.cubin")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    names = ("adam_kernel", "prune_gather_adam_kernel")
    spills, fn = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn is not None:
            spills[fn] = tuple(int(v) for v in m.groups())
            fn = None
    assert sorted(n for n in names if any(re.search(r"\d%s" % n, k) for k in spills)) == sorted(names), sorted(spills)
    bad = {k: v for k, v in spills.items() if v != (0, 0, 0)}
    assert not bad, bad
