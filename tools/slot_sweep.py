"""Developer aid (H100): per-kernel time of every layer-direction at every accumulator slot count the kernel
instantiations offer for it - the data the planner's time model (DGAN_COST_NS_PER_KB, DGAN_COST_OP_NS in
csrc/kernels_tc2.cuh) is fitted to.  Each direction is forced in turn to each slot count (dgan_debug_force_slots)
and timed with CUDA events around every launch (dgan_profile_*), graph replay off.
Usage: python tools/slot_sweep.py [mnist|celeba] [batch] [R] [L] [out.json]"""
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402

arch = sys.argv[1] if len(sys.argv) > 1 else "mnist"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
R = int(sys.argv[3]) if len(sys.argv) > 3 else 10
L = int(sys.argv[4]) if len(sys.argv) > 4 else 20
out_path = sys.argv[5] if len(sys.argv) > 5 else None

dev = torch.device("cuda", 0)
w = O.init_generator_weights(arch)
gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision="fp16", device=dev)
lib = gen.lib
lib.dgan_debug_force_slots.restype = ctypes.c_int
lib.dgan_debug_force_slots.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
lib.dgan_debug_slot_choices.restype = ctypes.c_int
lib.dgan_debug_slot_choices.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
imgs = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)


def timed():
    gen.reconstruct(imgs, R, 3, z_init_val=z0)            # plan, upload, warm up
    gen.profile_enable(True)
    gen.reconstruct(imgs, R, L, z_init_val=z0)
    torch.cuda.synchronize(dev)
    prof = gen.profile_read()
    gen.profile_enable(False)
    return {k["name"]: 1e3 * k["ms"] / k["launches"] for k in prof if k["launches"]}


rows = []
base = timed()
n_dirs = int(lib.dgan_profile_num_kinds(gen._handle)) - 1
names = [lib.dgan_profile_kind_name(gen._handle, d).decode() for d in range(n_dirs)]
for d in range(n_dirs):
    buf = (ctypes.c_int * 16)()
    n = lib.dgan_debug_slot_choices(gen._handle, d, buf, 16)
    for maxb in buf[:n]:
        assert lib.dgan_debug_force_slots(gen._handle, d, maxb) == 0, lib.dgan_last_error()
        us = timed()[names[d]]
        rows.append({"dir": d, "kernel": names[d], "maxb": maxb, "us": round(us, 2), "default_us": round(base[names[d]], 2)})
        print("%-22s maxb %d: %8.2f us (default plan %8.2f)" % (names[d], maxb, us, base[names[d]]), flush=True)
    assert lib.dgan_debug_force_slots(gen._handle, d, 0) == 0
gen.close()
if out_path:
    with open(out_path, "w") as f:
        json.dump({"arch": arch, "B": B, "R": R, "L": L, "gpu": torch.cuda.get_device_name(0), "rows": rows}, f, indent=1)
