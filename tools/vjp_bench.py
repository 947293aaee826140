"""Cost of a generator vector-Jacobian and Jacobian-vector product on one H100: CUDA-event medians of
NativeGenerator.forward, .vjp and .jvp, one L-step of reconstruct at the same latent rows ((time at L=20 - time at
L=10) / 10), the per-kernel times of one vjp / forward / L-step (dgan_profile_*, a separate pass), generator_jacobian of
20 MNIST and 8 CelebA images, and torch autograd / torch.func.jvp through the fp32 oracle generator (cuDNN, TF32 off) as
the do-it-yourself baselines.  Writes <out_dir>/vjp_bench.json.
Usage: python tools/vjp_bench.py OUT_DIR [--reps N] [--warmup N]"""
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

# (arch, images, restarts): MNIST 2560 latent rows (configs[1]'s batch), CelebA 1280
CASES = [("mnist", 256, 10), ("celeba", 640, 2)]
JACOBIAN_IMAGES = {"mnist": 20, "celeba": 8}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": out, "torch_name": torch.cuda.get_device_name(0)}


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def profile(gen, fn):
    """Per-kernel-kind ms per launch of one call of fn (plain launches, two events per launch)."""
    gen.profile_enable(True)
    fn()
    torch.cuda.synchronize()
    prof = gen.profile_read()
    gen.profile_enable(False)
    return {k["name"]: round(k["ms"] / k["launches"], 4) for k in prof if k["launches"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vjp_bench needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps, "warmup": a.warmup, "results": []}
    for arch, B, R in CASES:
        n = B * R
        w = O.init_generator_weights(arch)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        z = torch.tensor(O.sample_z0(n, 128)).to(dev)
        dy = torch.randn((n,) + tuple(x.shape[1:]), generator=torch.Generator().manual_seed(1)).to(dev)
        t = torch.randn((n, 128), generator=torch.Generator().manual_seed(2)).to(dev)
        zj = z[:JACOBIAN_IMAGES[arch]]
        for precision in ("fp16", "fp32"):
            gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision=precision,
                                          device=dev)
            r = {"arch": arch, "rows": n, "precision": precision}
            r["forward_ms"] = median_ms(lambda: gen.forward(z), a.reps, a.warmup)
            r["vjp_ms"] = median_ms(lambda: gen.vjp(z, dy), a.reps, a.warmup)
            r["jvp_ms"] = median_ms(lambda: gen.jvp(z, t), a.reps, a.warmup)
            r["jvp_over_forward"] = r["jvp_ms"] / r["forward_ms"]
            r["jacobian_images"] = len(zj)
            r["jacobian_ms"] = median_ms(lambda: gen.jacobian(zj), max(5, a.reps // 2), 2)
            t10 = median_ms(lambda: gen.reconstruct(x, R, 10, z_init_val=z), max(5, a.reps // 2), 2)
            t20 = median_ms(lambda: gen.reconstruct(x, R, 20, z_init_val=z), max(5, a.reps // 2), 2)
            r["reconstruct_L10_ms"], r["reconstruct_L20_ms"] = t10, t20
            r["l_step_ms"] = (t20 - t10) / 10.0
            r["vjp_over_lstep_plus_forward"] = r["vjp_ms"] / (r["l_step_ms"] + r["forward_ms"])
            r["profile_vjp_ms_per_launch"] = profile(gen, lambda: gen.vjp(z, dy))
            r["profile_forward_ms_per_launch"] = profile(gen, lambda: gen.forward(z))
            r["profile_reconstruct_L10_ms_per_launch"] = profile(gen, lambda: gen.reconstruct(x, R, 10, z_init_val=z))
            gen.close()
            print(json.dumps(r), flush=True)
            res["results"].append(r)
        # the baseline: torch autograd through the oracle generator, fp32 on the same GPU
        wt = {k: v.to(dev) for k, v in O.weights_to_torch(w, torch.float32).items()}

        def oracle_vjp():
            zt = z.detach().requires_grad_(True)
            torch.autograd.grad(O.generator_forward(arch, wt, zt), zt, dy)

        def oracle_fwd():
            with torch.no_grad():
                O.generator_forward(arch, wt, z)

        def oracle_jvp(zz, tt):
            with torch.no_grad():
                torch.func.jvp(lambda v: O.generator_forward(arch, wt, v), (zz,), (tt,))

        def oracle_jacobian():     # the same identity tangents as NativeGenerator.jacobian, all images in one call
            k = zj.shape[1]
            oracle_jvp(zj.repeat_interleave(k, dim=0), torch.eye(k, device=dev).repeat(len(zj), 1))

        r = {"arch": arch, "rows": n, "precision": "torch-fp32-cudnn (oracle.generator_forward, TF32 off)",
             "forward_ms": median_ms(oracle_fwd, a.reps, a.warmup), "vjp_ms": median_ms(oracle_vjp, a.reps, a.warmup),
             "jvp_ms": median_ms(lambda: oracle_jvp(z, t), a.reps, a.warmup), "jacobian_images": len(zj),
             "jacobian_ms": median_ms(oracle_jacobian, max(5, a.reps // 2), 2)}
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "vjp_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
