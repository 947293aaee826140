"""What the width rule costs on one H100: reconstruct() images/s at R=10, L=200 for generators at widths other than
latent_dim 128 / net_dim 64 (the rows of tests/test_gpu_widths.py) next to the default widths, on each precision that
serves the width, plus the per-kernel-kind times of one L=10 call (dgan_profile_*, a separate pass) and the padded
widths the handle stores.  MNIST at B=256, CelebA at B=128.  Reads the card's name, power limit and max SM clock from
nvidia-smi in the same run.  Writes <out_dir>/WIDTH_BENCH.json.
Usage: python tools/width_bench.py OUT_DIR [--reps N]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402

# (arch, latent_dim, net_dim, use_bn); the default widths first, as the yardstick
CASES = [("mnist", 128, 64, False), ("mnist", 100, 32, False), ("mnist", 128, 128, False),
         ("celeba", 128, 64, False), ("celeba", 200, 48, False), ("celeba", 64, 128, True)]
BATCH = {"mnist": 256, "celeba": 128}
R, L = 10, 200


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def padded_widths(lib, desc):
    """The widths the handle stores (the library's width rule): latent, 4 * net_dim, 2 * net_dim, net_dim."""
    out = (ctypes.c_int * 4)()
    lib.dgan_debug_padded_widths.restype = ctypes.c_int
    if lib.dgan_debug_padded_widths(ctypes.byref(desc), out) != 0:
        return None
    return dict(zip(("latent", "4*net_dim", "2*net_dim", "net_dim"), list(out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("width_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "R": R, "L": L, "reps": a.reps, "results": []}
    for arch, latent, nd, bn in CASES:
        B = BATCH[arch]
        w = O.init_generator_weights(arch, latent_dim=latent, net_dim=nd, use_bn=bn)
        x = torch.tensor(O.synthetic_images(arch, w, B, latent_dim=latent)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, latent)).to(dev)
        for precision in ("fp16", "fp32"):
            r = {"arch": arch, "latent_dim": latent, "net_dim": nd, "use_bn": bn, "precision": precision, "batch": B}
            try:
                gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], latent_dim=latent,
                                              net_dim=nd, use_bn=bn, precision=precision, device=dev)
            except RuntimeError as e:           # a width this precision does not serve
                r["refused"] = str(e)
                print(json.dumps(r), flush=True)
                res["results"].append(r)
                continue
            r["padded_widths"] = padded_widths(gen.lib, _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[arch], latent, nd,
                                                                           int(bn), _native.PRECISIONS[precision]))
            gen.reconstruct(x, R, L, z_init_val=z0)              # plans, captures the loop, warms up
            times = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                gen.reconstruct(x, R, L, z_init_val=z0)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) / 1e3)
            r["call_s"] = sorted(times)
            r["images_per_s"] = B / float(np.median(times))
            r["macs_per_row"] = gen.macs_per_row
            gen.profile_enable(True)
            gen.reconstruct(x, R, 10, z_init_val=z0)
            torch.cuda.synchronize()
            prof = gen.profile_read()
            gen.profile_enable(False)
            r["profile_L10_ms_per_launch"] = {k["name"]: round(k["ms"] / k["launches"], 4) for k in prof if k["launches"]}
            gen.close()
            print(json.dumps(r), flush=True)
            res["results"].append(r)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "WIDTH_BENCH.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
