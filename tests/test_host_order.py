"""CPU tests of the planner's item order (host code of the CUDA library; no GPU).  The default plans take a
layer-direction's items in bands of row pairs; dgan_debug_check_plans validates them, and the LPT plans, with
tc2_check_plan (every contribution exactly once, canonical order, ring safety, every item on exactly one CTA pair), and
dgan_debug_plan_order_stats reports what the order costs in balance and what it saves in working set."""
import ctypes

import pytest

ARCHS = {"mnist": 0, "celeba": 1}
TOLERANCE = 0.02          # TC2_BAND_TOLERANCE


def _lib():
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_check_plans.restype = ctypes.c_int
    lib.dgan_debug_check_plans.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_debug_plan_order_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_order_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_char_p, ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    return lib, _native


def _desc(arch, net_dim=64, use_bn=0):
    _, native = _lib()
    return native.dgan_desc(native.ABI_VERSION, ARCHS[arch], 128, net_dim, use_bn, 1)


def _order_stats(arch, n_rows, order, n_pairs=66, net_dim=64, use_bn=0):
    lib, _ = _lib()
    d = _desc(arch, net_dim, use_bn)
    buf = ctypes.create_string_buffer(1 << 16)
    n = lib.dgan_debug_plan_order_stats(ctypes.byref(d), n_rows, n_pairs, order, buf, len(buf))
    assert n > 0, (lib.dgan_last_error() or b"").decode()
    lines = [l.split(" | ") for l in buf.value.decode().strip().splitlines()]
    assert lines[0][-1] == "working set MB", lines[0]
    return {r[0]: r for r in lines[1:]}


def _check(arch, n_rows, n_pairs, net_dim=64, use_bn=0):
    lib, _ = _lib()
    d = _desc(arch, net_dim, use_bn)
    rc = lib.dgan_debug_check_plans(ctypes.byref(d), n_rows, n_pairs, 0)
    return rc, (lib.dgan_last_error() or b"").decode()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_banded_and_lpt_plans_pass_the_validator(arch):
    for n_rows in (1, 10, 256, 500, 1280, 2560, 5000, 5120):
        rc, msg = _check(arch, n_rows, 66)
        assert rc == 0, "n_rows=%d: %s" % (n_rows, msg)
    for n_pairs in (1, 3, 37, 66, 74):
        rc, msg = _check(arch, 2560 if arch == "mnist" else 640, n_pairs)
        assert rc == 0, "n_pairs=%d: %s" % (n_pairs, msg)


def test_banded_plans_pass_the_validator_for_random_sizes_and_sm_counts():
    pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=40, deadline=None)
    @given(st.sampled_from(["mnist", "celeba"]), st.integers(257, 6000), st.integers(1, 74), st.sampled_from([64, 32]),
           st.sampled_from([0, 1]))
    def run(arch, n_rows, n_pairs, net_dim, use_bn):
        rc, msg = _check(arch, n_rows, n_pairs, net_dim, use_bn)
        assert rc == 0 or "unsupported" in msg.lower(), (arch, n_rows, n_pairs, net_dim, use_bn, msg)

    run()


# configs[1] (2560 rows), CelebA B = 128 (1280 rows) and 512 MNIST images (5120 rows) on 66 CTA pairs
@pytest.mark.parametrize("arch,n_rows", [("mnist", 2560), ("celeba", 1280), ("mnist", 5120)])
def test_banded_makespan_is_within_the_tolerance_of_lpt(arch, n_rows):
    band = _order_stats(arch, n_rows, 1)
    lpt = _order_stats(arch, n_rows, 0)
    n_band = 0
    for name, r in band.items():
        lpt_us, order_us = float(r[3]), float(r[4])
        assert order_us <= lpt_us * (1 + TOLERANCE) + 0.05, (name, r)
        assert r[3] == lpt[name][3] and lpt[name][1] == "lpt" and lpt[name][4] == lpt[name][3], (name, r, lpt[name])
        # the order changes no item: the same bytes are staged
        assert r[5:8] == lpt[name][5:8], (name, r, lpt[name])
        if float(r[7]) < 9.4:          # TC2_BAND_MIN_INPUT: an input this small stays in L2 in any order
            assert r[1] == "lpt", (name, r)
        if r[1] != "lpt":
            n_band += 1
            assert r[1] in ("band+", "band-") and 1 <= int(r[2]) < n_rows // 256, (name, r)
    assert n_band >= 4, band
    # Generator.3 carries the largest tensors of the MNIST generator: both its directions are banded
    if arch == "mnist":
        assert band["Generator.3.fwd"][1] != "lpt" and band["Generator.3.bwd"][1] != "lpt", band


def test_band_direction_alternates_along_the_step():
    """Forward layers 0, 1, 2, .. then backward from the last layer down: consecutive directions walk their bands in
    opposite directions, so each starts on the row pairs its predecessor wrote last."""
    band = _order_stats("mnist", 5120, 1)
    seq = ["Linear.fwd", "Generator.2.fwd", "Generator.3.fwd", "last.fwd", "last.bwd", "Generator.3.bwd", "Generator.2.bwd",
           "Linear.bwd"]
    signs = {name: band[name][1][-1] for name in seq if band[name][1] != "lpt"}
    for i, a in enumerate(seq):
        for j, b in enumerate(seq):
            if a in signs and b in signs:
                assert (signs[a] == signs[b]) == ((i - j) % 2 == 0), (a, b, signs)

