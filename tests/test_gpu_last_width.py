"""GPU test (H100, -m gpu): the d(pre) block tensor of the last layer is stored at its real width, 16 * C_out channels
per 4x4 block instead of 64, so the fp16 workspace is smaller by n_blocks * n_pad * (64 - 16 * C_out) * 2 bytes."""
import ctypes

import pytest
import torch

from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

# dgan_workspace_bytes with the block tensor padded to 64 channels (fp16, latent 128, net_dim 64)
PADDED = {("mnist", False, 1, 1): 29113344, ("mnist", False, 256, 10): 291124224, ("mnist", False, 50, 10): 58225664,
          ("celeba", False, 1, 1): 146737152, ("celeba", False, 256, 10): 1467362304, ("celeba", False, 50, 10): 293473280,
          ("mnist", True, 1, 1): 57666560, ("mnist", True, 256, 10): 566776832, ("mnist", True, 50, 10): 114234368}


@pytest.mark.parametrize("arch,use_bn", [("mnist", False), ("celeba", False), ("mnist", True)])
def test_workspace_shrinks_by_the_block_tensor_padding(arch, use_bn):
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    w = O.init_generator_weights(arch, random_bias=True, use_bn=use_bn)
    gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], use_bn=use_bn, precision="fp16",
                                  device=dev)
    try:
        gen.lib.dgan_workspace_bytes.restype = ctypes.c_size_t
        n_blocks, c_out = (256, 3) if arch == "celeba" else (49, 1)
        for (a, bn, b, r), padded in PADDED.items():
            if (a, bn) != (arch, use_bn):
                continue
            n_pad = -(-b * r // 256) * 256
            got = int(gen.lib.dgan_workspace_bytes(gen._handle, b, r))
            assert got == padded - n_blocks * n_pad * (64 - 16 * c_out) * 2, (b, r, got, padded)
    finally:
        gen.close()
