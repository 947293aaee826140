"""CPU tests of the rounds that issue only their real ops (host code of the CUDA library; no GPU).

With 2 or 4 accumulator slots per round and 64-channel ops, the kernel issues a round's real ops alone and skips the
zero-tile ones; the plan
validator must then refuse a round without a real op, which would commit an empty wgmma group, and keep refusing a
zero-tile op that overwrites its accumulator."""
import ctypes

import pytest

from test_host import _check_plans
from test_host_slots import _stats

EMPTY_ROUND, FIRST_ZERO_TILE_OP = 14, 15       # dgan_debug_check_plans faults


def test_validator_rejects_a_round_without_a_real_op():
    rc, msg = _check_plans("mnist", 2560, mutate=EMPTY_ROUND)
    assert rc != 0 and msg.startswith("Generator.3.fwd:") and "round without a real op" in msg, (rc, msg)


def test_validator_rejects_a_zero_tile_op_that_overwrites():
    rc, msg = _check_plans("mnist", 2560, mutate=FIRST_ZERO_TILE_OP)
    assert rc != 0 and msg.startswith("Generator.3.fwd:") and "zero-tile op overwrites" in msg, (rc, msg)


@pytest.mark.parametrize("pass_name,fault", [("tangent", EMPTY_ROUND), ("tangent", FIRST_ZERO_TILE_OP),
                                             ("weighted", EMPTY_ROUND), ("weighted", FIRST_ZERO_TILE_OP)])
def test_the_other_passes_reject_the_same_faults(pass_name, fault):
    from defensegan_b200 import _native
    lib = _native.load_library()
    fn = getattr(lib, "dgan_debug_check_%s_plans" % pass_name)
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    desc = _native.dgan_desc(_native.ABI_VERSION, 0, 128, 64, 0, _native.PRECISIONS["fp16"])
    assert fn(ctypes.byref(desc), 2560, 66, 0) == 0, lib.dgan_last_error()
    assert fn(ctypes.byref(desc), 2560, 66, fault) != 0
    target = "Generator.3.jvp:" if pass_name == "tangent" else "last.fwd.w:"
    assert lib.dgan_last_error().decode().startswith(target), lib.dgan_last_error()


@pytest.mark.parametrize("arch,n_rows", [("mnist", 2560), ("celeba", 1280)])    # configs[1], CelebA B=128 x 10
def test_benchmarked_plans_pass_the_validator(arch, n_rows):
    for use_bn in (0, 1):
        rc, msg = _check_plans(arch, n_rows, use_bn=use_bn)
        assert rc == 0, (arch, use_bn, msg)


def _issue_stats(arch, n_rows):
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_plan_issue_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_issue_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_char_p,
                                                ctypes.c_int]
    desc = _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[arch], 128, 64, 0, _native.PRECISIONS["fp16"])
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.dgan_debug_plan_issue_stats(ctypes.byref(desc), n_rows, 66, buf, len(buf)) > 0
    return {r[0]: r for r in (l.split(" | ") for l in buf.value.decode().strip().splitlines()[1:])}


@pytest.mark.parametrize("arch,n_rows", [("mnist", 2560), ("celeba", 1280)])
def test_only_fixed_round_plans_issue_zero_tile_mmas(arch, n_rows):
    """Issued k16 MMAs are the real ones, plus the zero-tile ones only where the round is fixed (8 slots per round, or
    narrow ops); the plan statistics' k16 MMAs count every slot of every round, as the time model does, and the
    zero-tile share of them is what the other instantiations skip.  Plan statistics columns: 2 K, 7 MMAs (ops),
    10 zero-tile MMA %, 11 slots, 14 k16 MMAs."""
    plans, issue = _stats(arch, n_rows), _issue_stats(arch, n_rows)
    assert set(issue) == {name for name in plans if not name.startswith("total")}
    skipped = 0
    for name, r in issue.items():
        p = plans[name]
        k, ops, zero, slots, k16 = int(p[2]), int(p[7]), float(p[10]), int(p[11]), int(p[14])
        ksub = 4 if k % 64 == 0 else k // 16
        assert int(r[1]) == slots, (r, p)
        issued, skip = int(r[2]), int(r[3])
        assert issued + skip == k16 == ops * ksub, (r, p)
        if 1 < slots <= 4 and ksub == 4:
            # the zero-tile ops, to the rounding of the percentage
            assert abs(skip - k16 * zero / 100.0) <= k16 * 0.0005 + ksub, (r, p)
        else:
            assert skip == 0, (r, p)
        assert float(r[4]) <= float(p[12]) + 0.05, (r, p)      # estimated tensor time of the MMAs issued
        skipped += skip
    assert skipped > 0
    if arch == "mnist":
        # the last layer's forward issued 62,560 k16 MMAs per L-step when every slot of a round read an operand
        assert int(issue["last.fwd"][2]) < 62560 // 2, issue["last.fwd"]
