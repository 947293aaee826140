"""Adam against momentum in the projection, on one H100.

1. Speed: images/s of the Adam update against the momentum update (rec_optimizer "adam" / "momentum"), calls alternating
   repeat by repeat in one process with L2 flushed before each timed call (CUDA-event medians), on both precisions, for
     - bench.py's configs[1] (MNIST B = 256, R = 10, L = 200) and CelebA B = 128 (R = 10, L = 200);
     - one measured case: CelebA B = 128 with the 2x2 block average as a CSR operator;
     - one pruned case: MNIST B = 256 with "after 40 steps keep 2" ([(40, 2)]).
2. Effect: mean and worst final (min over restarts) loss at L = 50, 100 and 200 for a small rec_lr sweep per optimiser,
   fp16, R = 10.  By default on the seeded synthetic images of the other bench tools with the random-init (untrained)
   generator, which says nothing about a trained generator on real data; --ckpt (a generator.npz, read by
   defensegan_b200.weights.load_npz) and --images_npz (an .npz with an "images" array [N, H, W, C], already input-transformed) run
   it on those instead.
Records the card name and power limit.  Writes <out_dir>/adam_bench.json.
Usage: python tools/adam_bench.py OUT_DIR [--reps N] [--warmup N] [--skip_speed] [--skip_quality] [--arch mnist|celeba]
                                          [--ckpt W.npz] [--images_npz X.npz]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from defensegan_b200 import _native  # noqa: E402
from defensegan_b200 import weights as _weights  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402

ADAM = (0.9, 0.999, 1e-8)
# rec_lr of each optimiser in the timed runs: the reference's 10.0 for momentum; for Adam a step in z units
SPEED_LR = {"momentum": 10.0, "adam": 0.01}
# (name, arch, images, restarts, steps, kind): kind "image", "measured" (2x2 block average, CSR) or "pruned" ([(40, 2)])
SPEED_CASES = [("configs[1] MNIST", "mnist", 256, 10, 200, "image"), ("CelebA", "celeba", 128, 10, 200, "image"),
               ("CelebA block2 CSR", "celeba", 128, 10, 200, "measured"),
               ("MNIST pruned 40x2", "mnist", 256, 10, 200, "pruned")]
SWEEP = {"momentum": [1.0, 3.0, 10.0, 30.0], "adam": [0.001, 0.003, 0.01, 0.03, 0.1]}
SWEEP_STEPS = [50, 100, 200]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


_FLUSH = None


def flush_l2():
    """Overwrite 256 MB so that no operand of the previous call is left in the 50 MB L2."""
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    _FLUSH.fill_(1.0)


def timed(fn):
    flush_l2()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def make_gen(arch, weights, precision, dev):
    return _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in weights.values()], precision=precision,
                                   device=dev)


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
            opts = {"momentum": None, "adam": ADAM}

            def run(opt):
                if kind == "measured":
                    return gen.reconstruct_measured(y, op, R, L, SPEED_LR[opt], z_init_val=z0, adam=opts[opt])
                return gen.reconstruct(x, R, L, SPEED_LR[opt], z_init_val=z0, adam=opts[opt],
                                       prune=[(40, 2)] if kind == "pruned" else None)

            times = {k: [] for k in opts}
            launches = {}
            for i in range(a.warmup + a.reps):
                for opt in opts:
                    t = timed(lambda: run(opt))
                    launches[opt] = gen.last_launch_count
                    if i >= a.warmup:
                        times[opt].append(t)
            r = {"case": name, "arch": arch, "kind": kind, "precision": precision, "images": B, "restarts": R, "steps": L,
                 "launches": launches}
            for opt in opts:
                med = float(np.median(times[opt]))
                r[opt + "_ms"] = round(med, 3)
                r[opt + "_images_per_s"] = round(B / med * 1e3, 1)
                r[opt + "_spread_ms"] = [round(float(min(times[opt])), 3), round(float(max(times[opt])), 3)]
            r["adam_over_momentum_time"] = round(r["adam_ms"] / r["momentum_ms"], 4)
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
        imgs = O.synthetic_images(arch, w, a.quality_images)
        source += ", seeded synthetic images"
    B, R = imgs.shape[0], 10
    gen = make_gen(arch, w, "fp16", dev)
    x = torch.tensor(imgs).to(dev)
    z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
    out = {"arch": arch, "source": source, "images": B, "restarts": R, "precision": "fp16", "rows": []}
    for opt, lrs in SWEEP.items():
        for lr in lrs:
            for L in SWEEP_STEPS:
                _, loss, _ = gen.reconstruct(x, R, L, lr, z_init_val=z0, adam=ADAM if opt == "adam" else None,
                                             return_aux=True)
                lo = loss.double().cpu().numpy()
                row = {"optimizer": opt, "rec_lr": lr, "steps": L, "mean_loss": float(np.mean(lo)),
                       "worst_loss": float(np.max(lo)), "non_finite": int((~np.isfinite(lo)).sum())}
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
    ap.add_argument("--arch", default="mnist", choices=["mnist", "celeba"], help="the loss sweep's generator")
    ap.add_argument("--quality_images", type=int, default=64)
    ap.add_argument("--ckpt", default=None)
    ap.add_argument("--images_npz", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adam_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "adam": ADAM, "speed_lr": SPEED_LR}
    print(json.dumps(res["card"]), flush=True)
    if not a.skip_speed:
        res["speed"] = speed(a, dev)
    if not a.skip_quality:
        res["quality"] = quality(a, dev)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "adam_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
