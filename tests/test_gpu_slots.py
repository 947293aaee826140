"""GPU test (H100, -m gpu): every kernel instantiation the launch dispatch offers - each (N, accumulator slots per round,
epilogue, output type) - computes exactly what the planner's default choice computes.  Each layer-direction is forced
in turn to each slot count its (N, epilogue, output type) has; the reconstructions, losses and arg-min indices must be
bit-identical to the default plan's, because fewer slots only remove zero-tile MMAs (exact zeros) and every accumulator
keeps its summation order (k-chunk major, input pixel ascending)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


def _slot_choices(gen, d):
    lib = gen.lib
    lib.dgan_debug_slot_choices.restype = ctypes.c_int
    lib.dgan_debug_slot_choices.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    buf = (ctypes.c_int * 16)()
    n = lib.dgan_debug_slot_choices(gen._handle, d, buf, 16)
    return list(buf[:n]) if n > 0 else []


def _force(gen, d, maxb):
    lib = gen.lib
    lib.dgan_debug_force_slots.restype = ctypes.c_int
    lib.dgan_debug_force_slots.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    rc = lib.dgan_debug_force_slots(gen._handle, d, maxb)
    assert rc == 0, lib.dgan_last_error()


@pytest.mark.parametrize("arch,use_bn,B,R", [pytest.param("mnist", False, 6, 5, id="mnist-6-5"),
                                             pytest.param("celeba", False, 3, 4, id="celeba-3-4"),
                                             pytest.param("mnist", True, 6, 5, id="mnist-bn-6-5")])
def test_every_slot_count_reconstructs_bit_identically(arch, use_bn, B, R):
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    w = O.init_generator_weights(arch, random_bias=True, use_bn=use_bn)
    gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], use_bn=use_bn, precision="fp16",
                                  device=dev)
    try:
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=11)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, 128, seed=12)).to(dev)

        def run():
            rec, loss, idx = gen.reconstruct(imgs, R, 4, 10.0, z_init_val=z0, return_aux=True)
            return rec.cpu().numpy(), loss.cpu().numpy(), idx.cpu().numpy()

        want = run()
        n_dirs = int(gen.lib.dgan_profile_num_kinds(gen._handle)) - 1     # the last profile kind is the momentum update
        tried = 0
        # Most directions have a single instantiation, so forcing it reproduces the default plan.  Two instantiations
        # are compared on MNIST (Linear.bwd: 1 and 2 slots, last.fwd: 4 and 8) and one on CelebA (Linear.bwd).
        for d in range(n_dirs):
            choices = _slot_choices(gen, d)
            assert choices, d
            for maxb in choices:
                _force(gen, d, maxb)
                got = run()
                for a, b in zip(got, want):
                    np.testing.assert_array_equal(a, b, err_msg="direction %d, %d slots per round" % (d, maxb))
                tried += 1
            _force(gen, d, 0)
        assert tried > n_dirs          # at least one direction has a choice
        # a slot count without an instantiation is refused by name
        gen.lib.dgan_debug_force_slots.restype = ctypes.c_int
        assert gen.lib.dgan_debug_force_slots(gen._handle, 0, 3) != 0
        assert b"instantiation" in gen.lib.dgan_last_error()
    finally:
        gen.close()
