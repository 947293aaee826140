"""CPU tests of the width rule (host code of the CUDA library; no GPU).  A handle stores every channel width padded with
exact zeros - fp32 path: the next multiple of 64; fp16 path: the smallest of 64, 128 and 256, above that the next multiple
of 256 in column blocks of 256 channels - so any latent_dim and net_dim the fp16 path's envelope holds (latent_dim <= 256,
net_dim <= 128) is planned on tensor-core instantiations, and anything outside it is refused by name."""
import ctypes
import hashlib

import pytest

ARCHS = {"mnist": 0, "celeba": 1}
# (arch, latent_dim, net_dim, use_bn): the widths of the GPU tests and the envelope's corners
GRID = [("mnist", 100, 32, 0), ("mnist", 128, 128, 0), ("celeba", 200, 48, 0), ("celeba", 64, 128, 1), ("celeba", 64, 64, 1),
        ("mnist", 1, 1, 0), ("mnist", 256, 128, 1), ("celeba", 17, 13, 1), ("mnist", 65, 33, 1), ("celeba", 129, 97, 0)]


def _lib():
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_check_plans.restype = ctypes.c_int
    lib.dgan_debug_check_plans.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_debug_plan_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_char_p,
                                          ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    return lib, _native


def _desc(arch, latent, net_dim, use_bn, precision=1):
    from defensegan_b200 import _native
    return _native.dgan_desc(_native.ABI_VERSION, ARCHS[arch], latent, net_dim, use_bn, precision)


def _check(arch, latent, net_dim, use_bn, n_rows, n_pairs=66, mutate=0):
    lib, _ = _lib()
    d = _desc(arch, latent, net_dim, use_bn)
    rc = lib.dgan_debug_check_plans(ctypes.byref(d), n_rows, n_pairs, mutate)
    return rc, (lib.dgan_last_error() or b"").decode()


def _stats(arch, latent, net_dim, use_bn, n_rows, n_pairs=66):
    lib, _ = _lib()
    d = _desc(arch, latent, net_dim, use_bn)
    buf = ctypes.create_string_buffer(1 << 16)
    n = lib.dgan_debug_plan_stats(ctypes.byref(d), n_rows, n_pairs, buf, len(buf))
    assert n > 0, (lib.dgan_last_error() or b"").decode()
    return buf.value.decode()


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", GRID)
@pytest.mark.parametrize("n_rows", [1, 300, 2560])
def test_plans_at_padded_widths_pass_the_validator(arch, latent, net_dim, use_bn, n_rows):
    rc, msg = _check(arch, latent, net_dim, use_bn, n_rows)
    assert rc == 0, msg


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [("mnist", 100, 32, 0), ("celeba", 200, 48, 0)])
def test_validator_rejects_damaged_plans_at_padded_widths(arch, latent, net_dim, use_bn):
    """The fault injections of dgan_debug_check_plans are each reported at widths other than the default ones too."""
    for mutate in range(1, 14):
        rc, msg = _check(arch, latent, net_dim, use_bn, 2560, mutate=mutate)
        where = "last.bwd:" if mutate >= 12 else "Generator.3.fwd:"
        assert rc != 0 and msg.startswith(where), (mutate, rc, msg)


def test_plans_for_random_widths_sizes_and_sm_counts():
    pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=40, deadline=None)
    @given(st.sampled_from(["mnist", "celeba"]), st.integers(1, 3000), st.integers(1, 74), st.integers(1, 256),
           st.integers(1, 128), st.sampled_from([0, 1]))
    def run(arch, n_rows, n_pairs, latent, net_dim, use_bn):
        rc, msg = _check(arch, latent, net_dim, use_bn, n_rows, n_pairs=n_pairs)
        assert rc == 0, (arch, n_rows, n_pairs, latent, net_dim, use_bn, msg)

    run()


@pytest.mark.parametrize("latent,net_dim,what", [(128, 129, "unsupported net_dim 129: the fp16 path takes net_dim <= 128"),
                                                  (64, 256, "unsupported net_dim 256: the fp16 path takes net_dim <= 128"),
                                                  (257, 64, "unsupported latent_dim 257: the fp16 path takes latent_dim <= 256"),
                                                  (0, 64, "unsupported widths"), (128, -1, "unsupported widths")])
def test_widths_outside_the_fp16_envelope_are_refused_by_name(latent, net_dim, what):
    for arch in ARCHS:
        rc, msg = _check(arch, latent, net_dim, 0, 256)
        assert rc == -3 and msg.startswith(what), (arch, rc, msg)


@pytest.mark.parametrize("arch,net_dim,limit", [("celeba", 257, 256), ("mnist", 705, 704)])
def test_fp32_refuses_only_what_its_last_layer_cannot_hold(arch, net_dim, limit):
    """dgan_create checks the widths before it touches a device: the fp32 last layer keeps its filter and a band of input
    rows in shared memory (227 KB on an H100), which bounds net_dim; every smaller width is accepted."""
    lib, native = _lib()
    lib.dgan_create.restype = ctypes.c_int
    lib.dgan_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(native.dgan_desc),
                                ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_void_p]
    d = _desc(arch, 100, net_dim, 0, precision=0)
    n = lib.dgan_num_weights(ctypes.byref(d))
    arr = (ctypes.c_void_p * n)(*([1] * n))
    h = ctypes.c_void_p(0)
    assert lib.dgan_create(ctypes.byref(h), ctypes.byref(d), arr, n, None) == -3
    msg = lib.dgan_last_error().decode()
    assert msg.startswith("unsupported net_dim %d" % net_dim) and ("net_dim <= %d" % limit) in msg, msg


def _padded(arch, latent, net_dim, precision=1):
    lib, _ = _lib()
    lib.dgan_debug_padded_widths.restype = ctypes.c_int
    out = (ctypes.c_int * 4)()
    d = _desc(arch, latent, net_dim, 0, precision)
    assert lib.dgan_debug_padded_widths(ctypes.byref(d), out) == 0
    return list(out)


@pytest.mark.parametrize("latent,net_dim,want", [(100, 32, [128, 256, 64, 64]), (128, 128, [128, 512, 256, 128]),
                                                 (200, 48, [256, 256, 128, 64]), (64, 128, [64, 512, 256, 128]),
                                                 (128, 64, [128, 256, 128, 64]), (1, 1, [64, 256, 64, 64])])
def test_fp16_width_rule(latent, net_dim, want):
    """latent, 4 * net_dim, 2 * net_dim, net_dim: the smallest of 64 / 128 / 256, above 256 the next multiple of 256; the
    Linear's output at least 256 (its per-pixel bias is served by the N = 256 instantiations)."""
    assert _padded("mnist", latent, net_dim) == want


@pytest.mark.parametrize("latent,net_dim,want", [(100, 32, [128, 128, 64, 64]), (128, 64, [128, 256, 128, 64]),
                                                 (64, 128, [64, 512, 256, 128]), (1, 97, [64, 448, 256, 128])])
def test_fp32_width_rule(latent, net_dim, want):
    assert _padded("celeba", latent, net_dim, precision=0) == want


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", GRID)
def test_directions_carry_the_padded_widths(arch, latent, net_dim, use_bn):
    """N and K of every layer-direction are the padded widths: latent -> Linear, 4 * net_dim -> Generator.2,
    2 * net_dim -> Generator.3, net_dim -> the rest; the last layer's image side is not padded.  A layer-direction wider
    than 256 channels is one row per column block of 256, named by its channel range."""
    lat, c4, c2, c1 = _padded(arch, latent, net_dim)
    img = 48 if arch == "celeba" else 16
    logical = [("Linear.fwd", c4, lat), ("Linear.bwd", lat, c4), ("Generator.2.fwd", c2, c4), ("Generator.2.bwd", c4, c2),
               ("Generator.3.fwd", c1, c2), ("Generator.3.bwd", c2, c1)]
    if arch == "celeba":
        logical += [("Generator.5.fwd", c1, c1), ("Generator.5.bwd", c1, c1)]
    logical += [("last.fwd", img, c1), ("last.bwd", c1, img)]
    want = []
    for name, n, k in logical:
        want += [(name, n, k)] if n <= 256 else [("%s[%d:%d]" % (name, a, a + 256), 256, k) for a in range(0, n, 256)]
    rows = [l.split(" | ") for l in _stats(arch, latent, net_dim, use_bn, 256).strip().splitlines()[1:-1]]
    assert [(r[0], int(r[1]), int(r[2])) for r in rows] == want


# SHA-256 of the plan statistics (every layer-direction's N, K, window, items, slots, steps, MMAs, staged bytes, balance,
# epilogue) at the default widths, computed at the commit before the width rule: padding must not change them.
DEFAULT_PLAN_DIGESTS = {
    ("mnist", 2560): "f17f4085be74f67bfcbda6112c60459504c168a661df10ca65f9f4341657cb09",
    ("celeba", 1280): "1d4dcebda68825e7ce1b5c02c1324cff57f40edd301c835814afd3a96fa4c240",
}


@pytest.mark.parametrize("arch,n_rows", sorted(DEFAULT_PLAN_DIGESTS))
def test_default_width_plans_are_unchanged(arch, n_rows):
    got = hashlib.sha256(_stats(arch, 128, 64, 0, n_rows).encode()).hexdigest()
    assert got == DEFAULT_PLAN_DIGESTS[(arch, n_rows)]
