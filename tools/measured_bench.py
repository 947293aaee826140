"""Cost of the projection from linear measurements on one H100, all in one process:
  - images/s of NativeGenerator.reconstruct_measured with a Gaussian sketch at MNIST B = 256, R = 10, L = 200 for
    m in {100, 392, 784} and at CelebA B = 128, R = 10, L = 200 for m in {500, 2000}, and of the plain reconstruct at the
    same sizes, measured and plain calls alternating repeat by repeat with L2 flushed before each timed call (CUDA-event
    medians);
  - the same measured loop written the way a user would without it (generator_fn autograd through the vjp, torch matmuls,
    torch.optim.SGD with momentum), at a reduced L, reported per step;
  - the device time of the two measurement products (torch.profiler, CUDA activities, over dgan_loss_grad_measured calls)
    and their rate against the TF32 data-sheet figure (495 TFLOP/s dense, H100 SXM);
  - the card name and power limit.
Writes <out_dir>/measured_bench.json.
Usage: python tools/measured_bench.py OUT_DIR [--reps N] [--warmup N] [--precision fp16|fp32] [--user-steps N]"""
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

# (arch, images, restarts, steps, measurement counts)
CASES = [("mnist", 256, 10, 200, (100, 392, 784)), ("celeba", 128, 10, 200, (500, 2000))]
TF32_TFLOPS = 495.0


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


def user_loop(gen, y, a, z0, R, L, lr=10.0, momentum=0.7):
    """What a user writes today: generator_fn autograd, torch matmuls and torch momentum SGD on (1/m)||A G(z) - y||^2."""
    m = a.shape[0]
    z = z0.clone().requires_grad_(True)
    opt = torch.optim.SGD([z], lr=lr, momentum=momentum)
    y_rows = y.repeat_interleave(R, dim=0)
    for _ in range(L):
        opt.zero_grad(set_to_none=True)
        g = _native.generator(gen, z).reshape(z.shape[0], -1)
        loss = ((g @ a.t() - y_rows) ** 2).sum(dim=1) / m
        loss.sum().backward()
        opt.step()
    return z.detach()


def kernel_times(gen, y, a, z, R, calls=10):
    """Mean device time per call of each measurement product over dgan_loss_grad_measured calls (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    gen.loss_grad_measured(y, a, z, R)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            gen.loss_grad_measured(y, a, z, R)
        torch.cuda.synchronize()
    out = {"measure": 0.0, "adjoint": 0.0}
    for ka in prof.key_averages():
        if "measured_gemm_kernel" not in ka.key:          # <TC, 0>: the measurement product, <TC, 1>: the adjoint
            continue
        key = "measure" if "0>" in ka.key else "adjoint"
        out[key] += ka.device_time_total / 1e3 / calls    # us -> ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    ap.add_argument("--user-steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measured_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "warmup": args.warmup, "precision": args.precision, "results": []}
    for arch, B, R, L, ms in CASES:
        w = O.init_generator_weights(arch)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        hwc = x[0].numel()
        z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
        gen = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision=args.precision,
                                      device=dev)
        ops = {m: torch.tensor(MO.gaussian_operator(m, hwc, seed=m)).to(dev) for m in ms}
        ys = {m: x.reshape(B, -1) @ a.t() for m, a in ops.items()}
        calls = {"plain": lambda: gen.reconstruct(x, R, L, 10.0, z_init_val=z0)}
        for m in ms:
            calls["m%d" % m] = (lambda m=m: gen.reconstruct_measured(ys[m], ops[m], R, L, 10.0 * m / hwc, z_init_val=z0))
        times = {k: [] for k in calls}
        for i in range(args.warmup + args.reps):
            for name, fn in calls.items():
                t = timed(fn)
                if i >= args.warmup:
                    times[name].append(t)
        plain = float(np.median(times["plain"]))
        r = {"arch": arch, "images": B, "restarts": R, "steps": L, "precision": args.precision,
             "plain_ms": round(plain, 3), "plain_images_per_s": round(B / plain * 1e3, 1),
             "plain_spread_ms": [round(min(times["plain"]), 3), round(max(times["plain"]), 3)], "measured": []}
        for m in ms:
            t = times["m%d" % m]
            med = float(np.median(t))
            kt = kernel_times(gen, ys[m], ops[m], z0, R)
            flops = 2.0 * B * R * m * hwc                      # each product, algorithmic (unpadded m)
            r["measured"].append({
                "m": m, "ms": round(med, 3), "images_per_s": round(B / med * 1e3, 1),
                "spread_ms": [round(min(t), 3), round(max(t), 3)], "over_plain": round(med / plain, 4),
                "measure_product_ms": round(kt["measure"], 4), "adjoint_product_ms": round(kt["adjoint"], 4),
                "measure_product_tflops": round(flops / kt["measure"] / 1e9, 1) if kt["measure"] > 0 else None,
                "adjoint_product_tflops": round(flops / kt["adjoint"] / 1e9, 1) if kt["adjoint"] > 0 else None,
                "tf32_datasheet_tflops": TF32_TFLOPS})
        # the user-written loop at the largest m, a few steps, per step (after one warm-up step)
        m = ms[-1]
        user_loop(gen, ys[m], ops[m], z0, R, 1, lr=10.0 * m / hwc)
        tu = timed(lambda: user_loop(gen, ys[m], ops[m], z0, R, args.user_steps, lr=10.0 * m / hwc)) / args.user_steps
        tn = float(np.median(times["m%d" % m])) / L
        r["user_loop"] = {"m": m, "steps": args.user_steps, "ms_per_step": round(tu, 3),
                          "native_ms_per_step": round(tn, 3), "speedup": round(tu / tn, 2)}
        gen.close()
        print(json.dumps(r), flush=True)
        res["results"].append(r)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "measured_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
