"""Cost and effect of restart pruning on one H100: NativeGenerator.reconstruct on MNIST at configs[1] (B = 256, R = 10,
L = 200) and at batch 50, on the fp16 path, without pruning and with the schedules below, alternating call by call so
that clock and thermal drift fall on all of them alike.  CUDA-event median of each.  For each schedule, against the
unpruned call on the same seeded z0: the share of images whose chosen restart is unchanged and quantiles of
(pruned min loss / unpruned min loss).  Also the step time of a plain call at each stage's row count (R = keep), to say
where the time of a pruned call goes.  Records the card name and power limit.  Writes <out_dir>/prune_bench.json.

The images are seeded synthetic ones (oracle/defensegan_oracle.py synthetic_images, on the random-init generator), so
the agreement says nothing about a trained generator on real data; --ckpt (a generator.npz) with --images_npz (an .npz
whose "images" array is [N, 28, 28, 1], already input-transformed) runs the same on those.
Usage: python tools/prune_bench.py OUT_DIR [--reps N] [--warmup N] [--ckpt generator.npz --images_npz images.npz]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native  # noqa: E402
from defensegan_b200 import weights as _weights  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402

# (images, restarts, steps)
CASES = [(256, 10, 200), (50, 10, 200)]
SCHEDULES = {"none": None, "40x2": [(40, 2)], "20x5-60x2-120x1": [(20, 5), (60, 2), (120, 1)]}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def timed(fn, reps, warmup):
    """Median and range (ms) of CUDA-event timings of fn, after warmup calls."""
    t = []
    for i in range(warmup + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            t.append(e0.elapsed_time(e1))
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ckpt", default=None, help="generator.npz of a trained MNIST generator")
    ap.add_argument("--images_npz", default=None, help=".npz with 'images' [N, 28, 28, 1], input-transformed")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prune_bench needs a CUDA device")
    if (a.ckpt is None) != (a.images_npz is None):
        raise SystemExit("--ckpt and --images_npz go together")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "precision": "fp16", "results": []}
    sources = [("synthetic", None, None)]
    if a.ckpt is not None:
        sources.append(("checkpoint", a.ckpt, a.images_npz))
    for source, ckpt, images_npz in sources:
        w = _weights.load_npz(ckpt) if ckpt else O.init_generator_weights("mnist")
        ordered = _weights.validate_weights("mnist", w, 128, 64, False) if ckpt else list(w.values())
        gen = _native.NativeGenerator("mnist", [torch.as_tensor(np.asarray(v, dtype=np.float32)).to(dev) for v in ordered],
                                      precision="fp16", device=dev)
        for B, R, L in CASES:
            if images_npz:
                imgs = np.load(images_npz)["images"][:B].astype(np.float32)
                B = imgs.shape[0]
            else:
                imgs = O.synthetic_images("mnist", w, B)
            x = torch.tensor(imgs).to(dev)
            z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
            out = {}

            def run(prune):
                return gen.reconstruct(x, R, L, 10.0, z_init_val=z0, prune=prune, return_aux=True)

            times = {k: [] for k in SCHEDULES}
            for i in range(a.warmup + a.reps):
                for name, prune in SCHEDULES.items():
                    t = timed(lambda: run(prune), 1, 0)
                    if i >= a.warmup:
                        times[name] += t
            r = {"source": source, "images": B, "restarts": R, "steps": L}
            base = [t.clone() for t in run(None)]
            for name, prune in SCHEDULES.items():
                med = float(np.median(times[name]))
                r[name + "_ms"] = round(med, 3)
                r[name + "_images_per_s"] = round(B / med * 1e3, 1)
                r[name + "_spread_ms"] = [round(float(min(times[name])), 3), round(float(max(times[name])), 3)]
                if prune is None:
                    continue
                rec, loss, idx = run(prune)
                r[name + "_speedup"] = round(r["none_ms"] / med, 3)
                r[name + "_restart_agreement"] = round(float((idx == base[2]).float().mean()), 4)
                ratio = (loss / base[1]).double().cpu().numpy()
                r[name + "_loss_ratio_q"] = {q: round(float(np.quantile(ratio, q)), 5) for q in (0.0, 0.5, 0.9, 0.99, 1.0)}
            # where the time goes: the step time of a plain call at each stage's row count
            step = {}
            for keep in sorted({k for s in SCHEDULES.values() if s for _, k in s} | {R}):
                t = timed(lambda: gen.reconstruct(x, keep, L, 10.0, seed=1), a.reps, a.warmup)
                step[keep] = float(np.median(t)) / L
            r["step_ms_at_restarts"] = {str(k): round(v, 4) for k, v in step.items()}
            for name, prune in SCHEDULES.items():
                if prune is None:
                    continue
                its = [0] + [it for it, _ in prune] + [L]
                keeps = [R] + [k for _, k in prune]
                r[name + "_modelled_ms"] = round(sum((its[j + 1] - its[j]) * step[keeps[j]] for j in range(len(keeps))), 3)
            print(json.dumps(r), flush=True)
            res["results"].append(r)
        gen.close()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "prune_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
