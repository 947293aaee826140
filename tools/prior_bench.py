"""The latent prior (J = D + lambda ||z||^2) against the same call without it, on one H100.

1. Speed: images/s of the call without the prior (z_prior None) against lambda = 0.1, calls alternating repeat by repeat
   in one process with L2 flushed before each timed call (CUDA-event medians), on both precisions, R = 10, L = 200, for
   MNIST B = 256 (bench.py's configs[1]) and CelebA B = 128, each with
     - the image loss with momentum: on fp16 the prior runs the momentum update as a kernel of its own after the Linear
       backward instead of in its split-K tail (L - 1 launches more);
     - the image loss with Adam;
     - the 2x2 block average as a CSR operator, with momentum.
   The SM clock and power draw are sampled after each case.
2. Quality: how ||z|| of the chosen restart and the data term D move with lambda, fp16, R = 10, L = 200, on seeded
   synthetic S1 images (G(z*) plus noise) with the random-init (untrained) generator - which says nothing about a trained
   generator on real data: the image loss with momentum (rec_lr 10, the reference's) and with Adam (rec_lr 0.01), and
   the 4x4 block average (CSR) with Adam.  ||z|| is read back from the workspace (the final z of every restart), D is
   the fp64 data term of the returned reconstruction.
Records the card name and power limit.  Writes <out_dir>/prior_bench.json.
Usage: python tools/prior_bench.py OUT_DIR [--reps N] [--warmup N] [--skip_speed] [--skip_quality]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from adam_bench import card, make_gen, timed  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402

ADAM = (0.9, 0.999, 1e-8)
LAMBDA = 0.1
# (name, arch, images, restarts, steps)
SPEED_ARCHS = [("MNIST", "mnist", 256, 10, 200), ("CelebA", "celeba", 128, 10, 200)]
# kind: (loss, adam, rec_lr)
SPEED_KINDS = {"image momentum": ("image", None, 10.0), "image adam": ("image", ADAM, 0.01),
               "block2 CSR momentum": ("measured", None, 10.0)}
QUALITY_LAMBDAS = {"momentum": [0.0, 0.001, 0.01, 0.1], "adam": [0.0, 0.001, 0.01, 0.1, 1.0]}


def clocks():
    out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    return out


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
            op = dense.to_sparse_csr()
            for kind, (loss, adam, lr) in SPEED_KINDS.items():
                def run(lam):
                    if loss == "measured":
                        return gen.reconstruct_measured(y, op, R, L, lr, z_init_val=z0, adam=adam, z_prior=lam)
                    return gen.reconstruct(x, R, L, lr, z_init_val=z0, adam=adam, z_prior=lam)

                arms = {"none": None, "prior": LAMBDA}
                times = {k: [] for k in arms}
                launches = {}
                for i in range(a.warmup + a.reps):
                    for k, lam in arms.items():
                        t = timed(lambda: run(lam))
                        launches[k] = gen.last_launch_count
                        if i >= a.warmup:
                            times[k].append(t)
                r = {"case": "%s %s" % (name, kind), "arch": arch, "precision": precision, "images": B, "restarts": R,
                     "steps": L, "lambda": LAMBDA, "launches": launches, "clocks_sm_power": clocks()}
                for k in arms:
                    med = float(np.median(times[k]))
                    r[k + "_ms"] = round(med, 3)
                    r[k + "_images_per_s"] = round(B / med * 1e3, 1)
                    r[k + "_spread_ms"] = [round(float(min(times[k])), 3), round(float(max(times[k])), 3)]
                r["prior_over_none_time"] = round(r["prior_ms"] / r["none_ms"], 4)
                print(json.dumps(r), flush=True)
                out.append(r)
            gen.close()
            torch.cuda.empty_cache()
    return out


def final_z(gen, n_rows, m=0, nnz=-1):
    """The workspace's z [n_rows, latent] after an unpruned momentum or Adam call (iteration L-1 runs no update, so it is
    the z the returned loss was evaluated on).  The Adam layout is the momentum layout plus s, so z's offset is shared."""
    buf = ctypes.create_string_buffer(1 << 18)
    if m > 0:
        fn = gen.lib.dgan_debug_workspace_layout_measured_csr
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
        args = (gen._handle, n_rows, m, nnz, buf, len(buf))
    else:
        fn = gen.lib.dgan_debug_workspace_layout
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
        args = (gen._handle, n_rows, buf, len(buf))
    fn.restype = ctypes.c_int
    assert fn(*args) > 0
    f = next(ln.split() for ln in buf.value.decode().splitlines() if ln.split()[0] == "z")
    off, dims = int(f[2]), [int(v) for v in f[3:]]
    base = (gen._ws.data_ptr() + 1023) // 1024 * 1024 - gen._ws.data_ptr() + off
    torch.cuda.synchronize()
    z = gen._ws[base:base + dims[0] * dims[1] * 4].view(torch.float32).view(*dims)
    return z[:n_rows, :gen.latent_dim].double()


def quality(a, dev):
    arch, B, R, L = "mnist", a.quality_images, 10, 200
    w = O.init_generator_weights(arch)
    imgs = O.synthetic_images(arch, w, B, kind="S1")
    gen = make_gen(arch, w, "fp16", dev)
    x = torch.tensor(imgs).to(dev)
    z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
    box = torch.tensor(MO.block_average_operator(28, 28, 1, 4)).to(dev)
    y = x.reshape(B, -1).double() @ box.double().t()
    op = box.to_sparse_csr()
    out = {"arch": arch, "source": "random-init (untrained) generator, seeded synthetic S1 images", "images": B,
           "restarts": R, "steps": L, "precision": "fp16", "rows": []}
    cases = [("image momentum", None, 10.0, False), ("image adam", ADAM, 0.01, False),
             ("block4 CSR adam", ADAM, 0.01, True)]
    for name, adam, lr, measured in cases:
        for lam in QUALITY_LAMBDAS["adam" if adam else "momentum"]:
            if measured:
                rec, loss, idx = gen.reconstruct_measured(y.float(), op, R, L, lr, z_init_val=z0, adam=adam, z_prior=lam,
                                                          return_aux=True)
                zf = final_z(gen, B * R, m=box.shape[0], nnz=int(op.values().numel()))
                d = ((rec.reshape(B, -1).double() @ box.double().t() - y) ** 2).mean(dim=1)
            else:
                rec, loss, idx = gen.reconstruct(x, R, L, lr, z_init_val=z0, adam=adam, z_prior=lam, return_aux=True)
                zf = final_z(gen, B * R)
                d = ((rec.double() - x.double()) ** 2).mean(dim=(1, 2, 3))
            zc = zf.reshape(B, R, -1)[torch.arange(B), idx.long()]
            zn = zc.norm(dim=1)
            mse = ((rec.double() - x.double()) ** 2).mean(dim=(1, 2, 3))
            row = {"case": name, "lambda": lam, "rec_lr": lr, "mean_norm_z": float(zn.mean()),
                   "max_norm_z": float(zn.max()), "mean_D": float(d.mean()), "mean_mse_to_image": float(mse.mean()),
                   "mean_loss_J": float(loss.double().mean()), "non_finite": int((~torch.isfinite(loss)).sum())}
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
    ap.add_argument("--quality_images", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prior_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "adam": ADAM}
    print(json.dumps(res["card"]), flush=True)
    if not a.skip_speed:
        res["speed"] = speed(a, dev)
    if not a.skip_quality:
        res["quality"] = quality(a, dev)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "prior_bench.json"), "w") as f:
        json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
