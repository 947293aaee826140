"""GPU test (H100, -m gpu): the item order of the plans (dgan_debug_force_order: LPT over the whole batch, or row-pair
bands) decides only which CTA pair computes an item and when.  Every accumulator keeps its contributions and their order,
and the Linear backward's split-K partials are summed in part order, so reconstructions, losses and chosen restarts must
be bit-identical under both orders - for the plain, pruned and measured projections."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


def _force_order(gen, order):
    gen.lib.dgan_debug_force_order.restype = ctypes.c_int
    gen.lib.dgan_debug_force_order.argtypes = [ctypes.c_void_p, ctypes.c_int]
    rc = gen.lib.dgan_debug_force_order(gen._handle, order)
    assert rc == 0, gen.lib.dgan_last_error()


# B * R spans several row pairs of 256 rows, so the banded plans have more than one band
@pytest.mark.parametrize("arch,B,R", [pytest.param("mnist", 64, 10, id="mnist-64-10"),
                                      pytest.param("celeba", 32, 10, id="celeba-32-10")])
def test_item_order_does_not_change_results(arch, B, R):
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    w = O.init_generator_weights(arch, random_bias=True)
    gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision="fp16", device=dev)
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=21)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, 128, seed=22)).to(dev)
        hwc = x[0].numel()
        m = hwc // 2
        g = torch.Generator(device="cpu").manual_seed(23)
        a = (torch.randn(m, hwc, generator=g) / hwc ** 0.5).to(dev)
        y = x.reshape(B, -1) @ a.t()

        def run():
            outs = [gen.reconstruct(x, R, 6, 10.0, z_init_val=z0, return_aux=True),
                    gen.reconstruct(x, R, 6, 10.0, z_init_val=z0, return_aux=True, prune=[(2, 4), (4, 1)]),
                    gen.reconstruct_measured(y, a, R, 6, 10.0, z_init_val=z0, return_aux=True),
                    gen.reconstruct_measured(y, a, R, 6, 10.0, z_init_val=z0, return_aux=True, prune=[(3, 2)])]
            return [t.cpu().numpy() for o in outs for t in o]

        _force_order(gen, 0)
        lpt = run()
        _force_order(gen, 1)
        band = run()
        for i, (p, q) in enumerate(zip(lpt, band)):
            np.testing.assert_array_equal(p, q, err_msg="output %d" % i)
        assert gen.lib.dgan_debug_force_order(gen._handle, 2) != 0     # no such order
    finally:
        gen.close()
