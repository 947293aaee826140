"""CPU tests of the narrow last-layer backward (host code of the CUDA library; no GPU).  The d(pre) block tensor holds
only the 16 * C_out real channels of each 4x4 block (16 on MNIST, 48 on CelebA), and the last layer's backward stages
and multiplies 16-channel sub-tiles of it - one k16 MMA each - instead of 64-channel tiles that are 3/4 (MNIST) or 1/4
(CelebA) zeros."""
import ctypes

import pytest

from test_host import _check_plans

# The last layer's backward at configs[1] (MNIST, 2560 rows) and at 256 CelebA images x 10 restarts on 66 CTA pairs,
# planned with 64-channel ops (4 k16 MMAs each) over a K padded to 64: window, slots per round, ops, staged MB.
PADDED_LAST_BWD = {"mnist": ("1x4, 1x2", 4, 16160, 172.5), "celeba": ("1x4, 1x2", 4, 87040, 965.0)}
LAST_BWD = {"mnist": 7, "celeba": 9}          # row of last.bwd in the plan statistics


def _stats_at_window(arch, n_rows, d, maxb, shape):
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_plan_stats_window.restype = ctypes.c_int
    lib.dgan_debug_plan_stats_window.argtypes = [ctypes.POINTER(_native.dgan_desc)] + [ctypes.c_int] * 8 + \
        [ctypes.c_char_p, ctypes.c_int]
    desc = _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[arch], 128, 64, 0, _native.PRECISIONS["fp16"])
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.dgan_debug_plan_stats_window(ctypes.byref(desc), n_rows, 66, d, maxb, *shape, buf, len(buf)) > 0
    rows = [l.split(" | ") for l in buf.value.decode().strip().splitlines()[1:]]
    return {r[0]: r for r in rows}


@pytest.mark.parametrize("arch,use_bn", [("mnist", 0), ("celeba", 0), ("mnist", 1)])
@pytest.mark.parametrize("n_rows", [1, 300, 2560, 5120])
def test_narrow_plans_pass_the_validator(arch, use_bn, n_rows):
    rc, msg = _check_plans(arch, n_rows, use_bn=use_bn)
    assert rc == 0, msg


def test_validator_rejects_a_sub_tile_count_that_disagrees_with_the_instantiation():
    rc, msg = _check_plans("mnist", 2560, mutate=12)
    assert rc != 0 and msg.startswith("last.bwd:") and "k16 sub-tiles per op" in msg, (rc, msg)


def test_validator_rejects_a_second_k_chunk_of_a_narrow_operand():
    """A narrow K (16 * C_out < 64 channels) is a single k-chunk."""
    rc, msg = _check_plans("mnist", 2560, mutate=13)
    assert rc != 0 and msg.startswith("last.bwd:") and "out of range" in msg, (rc, msg)


@pytest.mark.parametrize("arch,cut", [("mnist", 4.0), ("celeba", 4.0 / 3.0)])
def test_last_bwd_stages_and_multiplies_only_real_channels(arch, cut):
    """At the padded plan's window and slot count, the narrow plan stages and issues at least `cut` times fewer bytes and
    k16 MMAs (MNIST: 16 of 64 channels, CelebA: 48 of 64)."""
    window, maxb, ops, mb = PADDED_LAST_BWD[arch]
    (wh, ww), (sy, sx) = [[int(v) for v in p.split("x")] for p in window.split(", ")]
    row = _stats_at_window(arch, 2560, LAST_BWD[arch], maxb, (wh, ww, sy, sx))["last.bwd"]
    assert row[3] == window and int(row[11]) == maxb, row
    assert int(row[2]) == (16 if arch == "mnist" else 48), row          # K: the real channels only
    assert float(row[8]) <= mb / cut + 0.05, (row[8], mb)
    assert int(row[14]) <= 4 * ops / cut, (row[14], 4 * ops)
