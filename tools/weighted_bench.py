"""Cost of the per-pixel weighted projection on one H100: NativeGenerator.reconstruct at configs[1] (MNIST, B = 256,
R = 10, L = 200) and CelebA (B = 128, R = 2, L = 200) on the fp16 path, unweighted, with weights of 1 and with a random
binary mask, the three alternating call by call so that clock and thermal drift fall on all of them alike.  CUDA-event
median of each.  Records the card name and power limit.  Writes <out_dir>/weighted_bench.json.
Usage: python tools/weighted_bench.py OUT_DIR [--reps N] [--warmup N] [--precision fp16|fp32]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402

# (arch, images, restarts, steps)
CASES = [("mnist", 256, 10, 200), ("celeba", 128, 2, 200)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("weighted_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "precision": a.precision, "results": []}
    for arch, B, R, L in CASES:
        w = O.init_generator_weights(arch)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
        ones = torch.ones_like(x)
        mask = (torch.rand(x.shape, generator=torch.Generator().manual_seed(1)) < 0.5).float().to(dev)
        gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision=a.precision,
                                      device=dev)
        variants = {"unweighted": None, "weights_1": ones, "binary_mask": mask}
        times = {k: [] for k in variants}
        for i in range(a.warmup + a.reps):
            for name, pw in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                gen.reconstruct(x, R, L, 10.0, z_init_val=z0, pixel_weights=pw)
                e1.record()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[name].append(e0.elapsed_time(e1))
        r = {"arch": arch, "images": B, "restarts": R, "steps": L, "precision": a.precision}
        for name, t in times.items():
            med = float(np.median(t))
            r[name + "_ms"] = round(med, 3)
            r[name + "_images_per_s"] = round(B / med * 1e3, 1)
            r[name + "_spread_ms"] = [round(float(min(t)), 3), round(float(max(t)), 3)]
        r["weights_1_over_unweighted"] = round(r["weights_1_ms"] / r["unweighted_ms"], 4)
        r["binary_mask_over_unweighted"] = round(r["binary_mask_ms"] / r["unweighted_ms"], 4)
        gen.close()
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "weighted_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
