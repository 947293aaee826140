"""Sparse deviations (fit G(z) + nu with an l1 penalty on nu) against the same call without them, on one H100.

1. Cost: images/s of each counterpart (sparse_dev None) against the call with deviations (tau = 0.1 at step = 1), calls
   alternating repeat by repeat in one process with L2 flushed before each timed call (CUDA-event medians), on both
   precisions, R = 10, L = 200, momentum at rec_lr 10, for MNIST B = 256 (bench.py's configs[1]) and CelebA B = 128:
     - the image loss: with deviations it leaves the fused last-layer epilogue for the measured loop;
     - a 5x5 Gaussian blur (ConvOperator, sigma 1.5);
     - the 2x2 block average as a CSR operator.
   The SM clock and power draw are sampled after each case.
2. Effect: seeded synthetic inputs with the random-init (untrained) generator - which says nothing about a trained
   generator on real data: x = G(z_t) with impulse noise on 2 % of the pixels (each set to the far end of the output
   range), z0 = z_t + 0.3 N(0, I), R = 2, L = 100, momentum at rec_lr 10, fp32 and fp16.  Prints the median
   ||G(z*) - G(z_t)|| without and with deviations (tau = a quarter of the output range, step 1) and the support precision
   and recall of nu* against the spiked pixels.
Records the card name and power limit.  Writes <out_dir>/sparse_dev_bench.json.
Usage: python tools/sparse_dev_bench.py OUT_DIR [--reps N] [--warmup N] [--skip_speed] [--skip_effect]"""
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
from prior_bench import clocks  # noqa: E402
from defensegan_b200.operators import ConvOperator  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402

TAU = 0.1
# (name, arch, images, restarts, steps)
SPEED_ARCHS = [("MNIST", "mnist", 256, 10, 200), ("CelebA", "celeba", 128, 10, 200)]
SPEED_KINDS = ["image", "conv blur5", "block2 CSR"]
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}


def speed(a, dev):
    out = []
    for precision in ("fp32", "fp16"):
        for name, arch, B, R, L in SPEED_ARCHS:
            w = O.init_generator_weights(arch)
            gen = make_gen(arch, w, precision, dev)
            x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
            z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
            dense = torch.tensor(MO.block_average_operator(*x.shape[1:], 2)).to(dev)
            y = x.reshape(B, -1) @ dense.t()
            csr = dense.to_sparse_csr()
            blur = ConvOperator.gaussian(5, 1.5)
            yb = blur(x.double()).float()
            dev_out = torch.empty_like(x)
            for kind in SPEED_KINDS:
                n = {"image": gen.hwc, "conv blur5": yb.shape[1], "block2 CSR": y.shape[1]}[kind]
                sd = (2 * TAU / n, 1.0)

                def run(s):
                    d = dev_out if s is not None else None
                    if kind == "image":
                        return gen.reconstruct(x, R, L, 10.0, z_init_val=z0, sparse_dev=s, deviation_out=d)
                    if kind == "conv blur5":
                        return gen.reconstruct_measured(yb, blur, R, L, 10.0, z_init_val=z0, sparse_dev=s,
                                                        deviation_out=d)
                    return gen.reconstruct_measured(y, csr, R, L, 10.0, z_init_val=z0, sparse_dev=s, deviation_out=d)

                arms = {"none": None, "sparse_dev": sd}
                times = {k: [] for k in arms}
                launches = {}
                for i in range(a.warmup + a.reps):
                    for k, s in arms.items():
                        t = timed(lambda: run(s))
                        launches[k] = gen.last_launch_count
                        if i >= a.warmup:
                            times[k].append(t)
                r = {"case": "%s %s" % (name, kind), "arch": arch, "precision": precision, "images": B, "restarts": R,
                     "steps": L, "l1": sd[0], "step": sd[1], "launches": launches, "clocks_sm_power": clocks()}
                for k in arms:
                    med = float(np.median(times[k]))
                    r[k + "_ms"] = round(med, 3)
                    r[k + "_images_per_s"] = round(B / med * 1e3, 1)
                    r[k + "_spread_ms"] = [round(float(min(times[k])), 3), round(float(max(times[k])), 3)]
                r["sparse_dev_over_none_time"] = round(r["sparse_dev_ms"] / r["none_ms"], 4)
                print(json.dumps(r), flush=True)
                out.append(r)
            gen.close()
            torch.cuda.empty_cache()
    return out


def effect(a, dev):
    rows = []
    B, R, L = a.effect_images, 2, 100
    for precision in ("fp32", "fp16"):
        for arch in ("mnist", "celeba"):
            w = O.init_generator_weights(arch)
            gen = make_gen(arch, w, precision, dev)
            g = torch.Generator().manual_seed(21)
            zt = torch.tensor(O.sample_z0(B, 128, seed=31)).to(dev)
            clean = gen.forward(zt).reshape((B,) + SHAPE[arch]).contiguous()
            lo, hi = (0.0, 1.0) if arch == "mnist" else (-1.0, 1.0)
            spiked = torch.rand(clean.shape, generator=g).to(dev) < 0.02
            far = torch.where(clean > (lo + hi) / 2, torch.full_like(clean, lo), torch.full_like(clean, hi))
            x = torch.where(spiked, far, clean)
            z0 = (zt.repeat_interleave(R, dim=0) + 0.3 * torch.randn(B * R, 128, generator=g).to(dev)).contiguous()
            tau = 0.25 * (hi - lo)
            sd = (2 * tau / gen.hwc, 1.0)
            plain = gen.reconstruct(x, R, L, 10.0, z_init_val=z0).clone()
            nu = torch.empty_like(x)
            robust = gen.reconstruct(x, R, L, 10.0, z_init_val=z0, sparse_dev=sd, deviation_out=nu).clone()
            e0 = (plain - clean).reshape(B, -1).norm(dim=1)
            e1 = (robust - clean).reshape(B, -1).norm(dim=1)
            on = nu != 0
            tp = float((on & spiked).sum())
            row = {"arch": arch, "precision": precision, "images": B, "restarts": R, "steps": L, "tau": tau,
                   "l1": sd[0], "step": sd[1], "spiked_fraction": float(spiked.double().mean()),
                   "median_err_without": float(e0.median()), "median_err_with": float(e1.median()),
                   "images_better_with": int((e1 < e0).sum()),
                   "support_precision": tp / max(float(on.sum()), 1.0), "support_recall": tp / float(spiked.sum()),
                   "source": "random-init (untrained) generator, seeded synthetic inputs"}
            print(json.dumps(row), flush=True)
            rows.append(row)
            gen.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--skip_speed", action="store_true")
    ap.add_argument("--skip_effect", action="store_true")
    ap.add_argument("--effect_images", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sparse_dev_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup}
    print(json.dumps(res["card"]), flush=True)
    if not a.skip_speed:
        res["speed"] = speed(a, dev)
    if not a.skip_effect:
        res["effect"] = effect(a, dev)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "sparse_dev_bench.json"), "w") as f:
        json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
