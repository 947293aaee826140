"""CPU tests of the accumulator-slot choice of the tensor-core planner (host code of the CUDA library; no GPU)."""
import ctypes

from test_host import _check_plans


def _stats(arch, n_rows, force_dir=-1, force_maxb=0):
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_plan_stats_slots.restype = ctypes.c_int
    lib.dgan_debug_plan_stats_slots.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    desc = _native.dgan_desc(_native.ABI_VERSION, 0 if arch == "mnist" else 1, 128, 64, 0, 1)
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.dgan_debug_plan_stats_slots(ctypes.byref(desc), n_rows, 66, force_dir, force_maxb, buf, len(buf)) > 0
    rows = [l.split(" | ") for l in buf.value.decode().strip().splitlines()[1:]]
    return {r[0]: r for r in rows}


def test_validator_rejects_a_slot_count_without_an_instantiation():
    rc, msg = _check_plans("mnist", 2560, mutate=10)
    assert rc != 0 and msg.startswith("Generator.3.fwd:") and "instantiation" in msg, (rc, msg)


def test_validator_rejects_records_that_disagree_with_the_plans_slot_count():
    """The launch dispatches on the plan's slot count and the kernel decodes the MMA records with it."""
    rc, msg = _check_plans("mnist", 2560, mutate=11)
    assert rc != 0 and msg.startswith("Generator.3.fwd:") and "disagrees with the plan" in msg, (rc, msg)


def test_planner_cuts_zero_tile_mmas_at_configs1():
    """configs[1]: the slot count is chosen per layer-direction.  Linear.bwd (one accumulator per window) runs on one
    slot and issues no zero-tile MMA; Generator.3.fwd and the last layer's forward issue far fewer than with the most
    slots (52 % and 72 % zero-tile MMAs before the choice existed)."""
    by = _stats("mnist", 2560)
    zero, slots, mmas = (lambda n: float(by[n][10])), (lambda n: int(by[n][11])), (lambda n: int(by[n][7]))
    assert slots("Linear.bwd") == 1 and zero("Linear.bwd") == 0.0
    assert zero("Generator.3.fwd") < 40.0 and zero("last.fwd") < 60.0
    assert float(by["total staged MB per L-step"][1]) < 1900.0
    # forcing the most slots reproduces the larger MMA counts: the choice is the planner's
    assert mmas("Linear.bwd") < int(_stats("mnist", 2560, 1, 2)["Linear.bwd"][7])
    assert mmas("last.fwd") < int(_stats("mnist", 2560, 6, 8)["last.fwd"][7])
