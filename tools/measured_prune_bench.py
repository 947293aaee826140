"""Cost and effect of restart pruning in the projection from linear measurements on one H100:
NativeGenerator.reconstruct_measured on the fp16 path at R = 10, L = 200 for
  - MNIST B = 256: a dense Gaussian sketch at m = 392 and the 2x2 block average as CSR;
  - CelebA B = 128: a dense Gaussian sketch at m = 500, the 2x2 block average as CSR and 4096-pixel subsampling as CSR;
without pruning and with the schedules below, calls alternating repeat by repeat with L2 flushed before each timed call
(CUDA-event medians).  For each schedule, against the unpruned call on the same seeded z0: images/s and the speedup, the
share of images whose chosen restart is unchanged and quantiles of (pruned min loss / unpruned min loss), as
tools/prune_bench.py reports them for the image loss.  Also the step time of an unpruned measured call at each stage's
row count (R = keep) and the sum-of-stages estimate it gives for each schedule, to say where the time of a pruned call
goes.  Records the card name and power limit.  Writes <out_dir>/measured_prune_bench.json.

The images are seeded synthetic ones on the random-init generator, so the agreement says nothing about a trained
generator on real data.
Usage: python tools/measured_prune_bench.py OUT_DIR [--reps N] [--warmup N] [--precision fp16|fp32]"""
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
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402
import sparse_operators as SO  # noqa: E402

SHAPES = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
# (arch, images, restarts, steps, [(operator name, passed as CSR)])
CASES = [("mnist", 256, 10, 200, [("gauss392", False), ("block2", True)]),
         ("celeba", 128, 10, 200, [("gauss500", False), ("block2", True), ("sub4096", True)])]
SCHEDULES = {"none": None, "40x2": [(40, 2)], "20x5-60x2-120x1": [(20, 5), (60, 2), (120, 1)]}


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


def operator(arch, name):
    h, w, c = SHAPES[arch]
    hwc = h * w * c
    if name == "block2":
        return MO.block_average_operator(h, w, c, 2)
    if name.startswith("sub"):
        return SO.subsample_operator(int(name[3:]), hwc, seed=1)
    m = int(name[5:])
    return MO.gaussian_operator(m, hwc, seed=m)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measured_prune_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "precision": a.precision, "results": []}
    for arch, B, R, L, ops in CASES:
        w = O.init_generator_weights(arch)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
        gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision=a.precision,
                                      device=dev)
        for name, as_csr in ops:
            a_np = operator(arch, name)
            m, hwc = a_np.shape
            lr = 10.0 * min(1.0, 4.0 * m / hwc)
            dense = torch.tensor(a_np).to(dev)
            y = x.reshape(B, -1) @ dense.t()
            op = dense.to_sparse_csr() if as_csr else dense

            def run(prune, rr=R, z=z0):
                return gen.reconstruct_measured(y, op, rr, L, lr, z_init_val=z, prune=prune, return_aux=True)

            times = {k: [] for k in SCHEDULES}
            for i in range(a.warmup + a.reps):
                for sname, prune in SCHEDULES.items():
                    t = timed(lambda: run(prune))
                    if i >= a.warmup:
                        times[sname].append(t)
            r = {"arch": arch, "operator": name, "csr": as_csr, "m": m, "images": B, "restarts": R, "steps": L,
                 "precision": a.precision}
            base = [t.clone() for t in run(None)]
            for sname, prune in SCHEDULES.items():
                med = float(np.median(times[sname]))
                r[sname + "_ms"] = round(med, 3)
                r[sname + "_images_per_s"] = round(B / med * 1e3, 1)
                r[sname + "_spread_ms"] = [round(float(min(times[sname])), 3), round(float(max(times[sname])), 3)]
                if prune is None:
                    continue
                _, loss, idx = run(prune)
                r[sname + "_speedup"] = round(r["none_ms"] / med, 3)
                r[sname + "_restart_agreement"] = round(float((idx == base[2]).float().mean()), 4)
                ratio = (loss / base[1]).double().cpu().numpy()
                r[sname + "_loss_ratio_q"] = {q: round(float(np.quantile(ratio, q)), 5) for q in (0.0, 0.5, 0.9, 0.99, 1.0)}
            # where the time goes: the step time of an unpruned measured call at each stage's row count
            step = {}
            for keep in sorted({k for s in SCHEDULES.values() if s for _, k in s} | {R}):
                zk = z0.view(B, R, -1)[:, :keep].reshape(B * keep, -1).contiguous()
                t = []
                for i in range(a.warmup + a.reps):
                    ti = timed(lambda: run(None, keep, zk))
                    if i >= a.warmup:
                        t.append(ti)
                step[keep] = float(np.median(t)) / L
            r["step_ms_at_restarts"] = {str(k): round(v, 4) for k, v in step.items()}
            for sname, prune in SCHEDULES.items():
                if prune is None:
                    continue
                its = [0] + [it for it, _ in prune] + [L]
                keeps = [R] + [k for _, k in prune]
                r[sname + "_modelled_ms"] = round(sum((its[j + 1] - its[j]) * step[keeps[j]] for j in range(len(keeps))), 3)
            print(json.dumps(r), flush=True)
            res["results"].append(r)
            del dense, op
            gen._ws = None
            torch.cuda.empty_cache()
        gen.close()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "measured_prune_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
