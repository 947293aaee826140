"""The Huber data term against the squared error in the projection, on one H100.

1. Speed: images/s of the squared error against the Huber loss at delta = +inf and at delta = 0.1, calls alternating
   repeat by repeat in one process with L2 flushed before each timed call (CUDA-event medians), on both precisions, for
     - bench.py's configs[1] (MNIST B = 256, R = 10, L = 200) and CelebA B = 128 (R = 10, L = 200);
     - one measured case: CelebA B = 128 with the 2x2 block average as a CSR operator;
     - one pruned case: MNIST B = 256 with "after 40 steps keep 2" ([(40, 2)]).
2. Quality: S1 images (G(z*) plus noise) with salt-and-pepper corruption - a share p of the pixels set to either end of
   the generator's range - for p in {0, 0.05, 0.2}; the mean squared error of the reconstruction against the uncorrupted
   image for delta in {inf, 0.3, 0.1, 0.03}, with momentum (rec_lr 10, the reference's) and Adam (rec_lr 0.01), fp16,
   R = 10, L = 200.  By default on the seeded synthetic images with the random-init (untrained) generator, which says
   nothing about a trained generator on real data; --ckpt (a generator.npz, read by defensegan_b200.weights.load_npz) and
   --images_npz (an .npz with an "images" array [N, H, W, C], already input-transformed) run it on those instead.
Records the card name and power limit.  Writes <out_dir>/huber_bench.json.
Usage: python tools/huber_bench.py OUT_DIR [--reps N] [--warmup N] [--skip_speed] [--skip_quality] [--arch mnist|celeba]
                                           [--ckpt W.npz] [--images_npz X.npz]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from adam_bench import card, make_gen, timed  # noqa: E402
from defensegan_b200 import weights as _weights  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402

ADAM = (0.9, 0.999, 1e-8)
# the squared error (None) against the Huber loss at +inf (the same arithmetic path, nothing clipped) and at 0.1
SPEED_DELTAS = {"squared": None, "huber_inf": float("inf"), "huber_0.1": 0.1}
# (name, arch, images, restarts, steps, kind): kind "image", "measured" (2x2 block average, CSR) or "pruned" ([(40, 2)])
SPEED_CASES = [("configs[1] MNIST", "mnist", 256, 10, 200, "image"), ("CelebA", "celeba", 128, 10, 200, "image"),
               ("CelebA block2 CSR", "celeba", 128, 10, 200, "measured"),
               ("MNIST pruned 40x2", "mnist", 256, 10, 200, "pruned")]
QUALITY_P = [0.0, 0.05, 0.2]
QUALITY_DELTAS = [float("inf"), 0.3, 0.1, 0.03]
QUALITY_LR = {"momentum": 10.0, "adam": 0.01}


def salt_and_pepper(x, arch, p, seed=5):
    """x with a share p of its pixels set to either end of the generator's range, at random (seeded)."""
    g = torch.Generator().manual_seed(seed)
    lo = 0.0 if arch == "mnist" else -1.0
    hit = (torch.rand(x.shape, generator=g) < p).to(x.device)
    val = torch.where(torch.rand(x.shape, generator=g) < 0.5, lo, 1.0).to(x.device)
    return torch.where(hit, val, x)


def speed(a, dev):
    out = []
    for precision in ("fp32", "fp16"):
        for name, arch, B, R, L, kind in SPEED_CASES:
            w = O.init_generator_weights(arch)
            gen = make_gen(arch, w, precision, dev)
            x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
            z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
            if kind == "measured":
                dense = torch.tensor(MO.block_average_operator(*x.shape[1:], 2)).to(dev)
                y = x.reshape(B, -1) @ dense.t()
                op = dense.to_sparse_csr()

            def run(delta):
                if kind == "measured":
                    return gen.reconstruct_measured(y, op, R, L, 10.0, z_init_val=z0, huber_delta=delta)
                return gen.reconstruct(x, R, L, 10.0, z_init_val=z0, huber_delta=delta,
                                       prune=[(40, 2)] if kind == "pruned" else None)

            times = {k: [] for k in SPEED_DELTAS}
            launches = {}
            for i in range(a.warmup + a.reps):
                for k, delta in SPEED_DELTAS.items():
                    t = timed(lambda: run(delta))
                    launches[k] = gen.last_launch_count
                    if i >= a.warmup:
                        times[k].append(t)
            r = {"case": name, "arch": arch, "kind": kind, "precision": precision, "images": B, "restarts": R, "steps": L,
                 "launches": launches}
            for k in SPEED_DELTAS:
                med = float(np.median(times[k]))
                r[k + "_ms"] = round(med, 3)
                r[k + "_images_per_s"] = round(B / med * 1e3, 1)
                r[k + "_spread_ms"] = [round(float(min(times[k])), 3), round(float(max(times[k])), 3)]
            for k in ("huber_inf", "huber_0.1"):
                r[k + "_over_squared_time"] = round(r[k + "_ms"] / r["squared_ms"], 4)
            print(json.dumps(r), flush=True)
            out.append(r)
            gen.close()
            torch.cuda.empty_cache()
    return out


def quality(a, dev):
    arch = a.arch
    if a.ckpt:
        w = _weights.load_npz(a.ckpt)
        w = dict(zip(w.keys(), _weights.validate_weights(arch, w, 128, 64, False)))
        source = "checkpoint %s" % os.path.basename(a.ckpt)
    else:
        w = O.init_generator_weights(arch)
        source = "random-init (untrained) generator"
    if a.images_npz:
        imgs = np.load(a.images_npz)["images"][:a.quality_images].astype(np.float32)
        source += ", images from %s" % os.path.basename(a.images_npz)
    else:
        imgs = O.synthetic_images(arch, w, a.quality_images, kind="S1")
        source += ", seeded synthetic S1 images"
    B, R, L = imgs.shape[0], 10, 200
    gen = make_gen(arch, w, "fp16", dev)
    clean = torch.tensor(imgs).to(dev)
    z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
    out = {"arch": arch, "source": source, "images": B, "restarts": R, "steps": L, "precision": "fp16", "rec_lr": QUALITY_LR,
           "rows": []}
    for p in QUALITY_P:
        x = salt_and_pepper(clean, arch, p)
        for opt, lr in QUALITY_LR.items():
            for delta in QUALITY_DELTAS:
                rec = gen.reconstruct(x, R, L, lr, z_init_val=z0, adam=ADAM if opt == "adam" else None, huber_delta=delta)
                mse = ((rec.double() - clean.double()) ** 2).mean(dim=(1, 2, 3)).cpu().numpy()
                row = {"p": p, "optimizer": opt, "delta": delta, "mse_to_clean": float(np.mean(mse)),
                       "worst_mse_to_clean": float(np.max(mse)), "non_finite": int((~np.isfinite(mse)).sum())}
                print(json.dumps(row), flush=True)
                out["rows"].append(row)
    gen.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip_speed", action="store_true")
    ap.add_argument("--skip_quality", action="store_true")
    ap.add_argument("--arch", default="mnist", choices=["mnist", "celeba"], help="the quality sweep's generator")
    ap.add_argument("--quality_images", type=int, default=64)
    ap.add_argument("--ckpt", default=None)
    ap.add_argument("--images_npz", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("huber_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "adam": ADAM}
    print(json.dumps(res["card"]), flush=True)
    if not a.skip_speed:
        res["speed"] = speed(a, dev)
    if not a.skip_quality:
        res["quality"] = quality(a, dev)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "huber_bench.json"), "w") as f:
        json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
