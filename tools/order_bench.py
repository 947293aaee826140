"""Item order A/B on one H100: NativeGenerator.reconstruct on the fp16 path with every layer-direction planned in the LPT
order and in the banded order (dgan_debug_force_order), one handle per order, alternating call by call so that clock
and thermal drift fall on both alike.  Workloads: configs[1] (MNIST B = 256, R = 10, L = 200), CelebA B = 128 (configs[3])
and MNIST B = 512 (the per-GPU share of configs[4]).  Per call: L2 flushed (a 256 MB buffer zeroed before it), CUDA-event
time of the whole call.  Then the per-kernel CUDA-event pass (dgan_profile_*), alternating too.  Also checks that both
orders return bit-identical reconstructions, losses and chosen restarts.  Records the card name and power limit.
Writes <out_dir>/order_bench.json.
Usage: python tools/order_bench.py OUT_DIR [--reps N] [--warmup N] [--profile_reps N]"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402

CASES = [("configs[1]", "mnist", 256, 10, 200), ("CelebA B=128", "celeba", 128, 10, 200),
         ("MNIST 512 images", "mnist", 512, 10, 200)]
ORDERS = {"lpt": 0, "band": 1}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def force_order(gen, order):
    gen.lib.dgan_debug_force_order.restype = ctypes.c_int
    gen.lib.dgan_debug_force_order.argtypes = [ctypes.c_void_p, ctypes.c_int]
    rc = gen.lib.dgan_debug_force_order(gen._handle, order)
    if rc != 0:
        raise RuntimeError(gen.lib.dgan_last_error())


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile_reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("order_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "precision": "fp16", "results": []}
    for label, arch, B, R, L in CASES:
        w = O.init_generator_weights(arch)
        gens = {}
        for name, order in ORDERS.items():
            gens[name] = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision="fp16",
                                                 device=dev)
            force_order(gens[name], order)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
        outs, times = {}, {n: [] for n in ORDERS}
        for i in range(a.warmup + a.reps):
            for name in (ORDERS if i % 2 == 0 else reversed(list(ORDERS))):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rec, loss, idx = gens[name].reconstruct(x, R, L, 10.0, z_init_val=z0, return_aux=True)
                e1.record()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[name].append(e0.elapsed_time(e1))
                outs[name] = (rec.cpu().numpy(), loss.cpu().numpy(), idx.cpu().numpy())
        identical = all(np.array_equal(p, q) for p, q in zip(outs["lpt"], outs["band"]))
        kernels = {n: {} for n in ORDERS}
        for i in range(a.profile_reps):
            for name in (ORDERS if i % 2 == 0 else reversed(list(ORDERS))):
                g = gens[name]
                g.profile_enable(True)
                g.reconstruct(x, R, L, 10.0, z_init_val=z0)
                torch.cuda.synchronize()
                for k in g.profile_read():
                    if k["launches"]:
                        kernels[name].setdefault(k["name"], []).append(1e3 * k["ms"] / k["launches"])
                g.profile_enable(False)
        row = {"case": label, "arch": arch, "B": B, "R": R, "L": L, "bit_identical": identical,
               "call_ms": {n: spread(t) for n, t in times.items()},
               "images_per_s": {n: B / (statistics.median(t) / 1e3) for n, t in times.items()},
               "kernel_us": {n: {k: spread(v) for k, v in ks.items()} for n, ks in kernels.items()}}
        res["results"].append(row)
        print("%-18s identical=%s  call ms lpt %.2f [%.2f-%.2f]  band %.2f [%.2f-%.2f]" % (
            label, identical, *(row["call_ms"][n][s] for n in ORDERS for s in ("median", "min", "max"))))
        for k in kernels["lpt"]:
            lp, bd = row["kernel_us"]["lpt"][k], row["kernel_us"]["band"].get(k)
            if bd is not None:
                print("    %-24s lpt %8.1f [%7.1f-%7.1f]  band %8.1f [%7.1f-%7.1f] us" % (
                    k, lp["median"], lp["min"], lp["max"], bd["median"], bd["min"], bd["max"]))
        for g in gens.values():
            g.close()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "order_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
