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
With --sparse instead: sparse operators (a 2x2 block average, a full-resolution 5 x 5 blur, pixel subsampling at two m)
at MNIST B = 256 and CelebA B = 128, R = 10, L = 200, passed dense and as CSR; plain, dense and CSR calls alternate
repeat by repeat.  Reports images/s of each call, the device time of the CSR products (torch.profiler) with their
algorithmic bytes over it as a share of 3.35 TB/s (HBM3, H100 SXM data sheet), and the workspace bytes of both calls.
A dense call that does not fit in memory is reported as not run.  The block averages and the blur also run as a
ConvOperator (the stencil products of dgan_reconstruct_measured_conv), timed in the same alternation, and two more rows
run plain and convolution calls only: a 4x box downsample and per-image random 9 x 9 motion-blur kernels.  The product
times of the CSR and convolution calls are each set against the same byte count - G or r read once, r or dy written
once - as a share of 3.35 TB/s.  Writes <out_dir>/measured_bench_sparse.json.
Usage: python tools/measured_bench.py OUT_DIR [--reps N] [--warmup N] [--precision fp16|fp32] [--user-steps N] [--sparse]"""
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
from defensegan_b200 import _native  # noqa: E402
from oracle import defensegan_oracle as O  # noqa: E402
import measured_oracle as MO  # noqa: E402
import sparse_operators as SO  # noqa: E402

# (arch, images, restarts, steps, measurement counts)
CASES = [("mnist", 256, 10, 200, (100, 392, 784)), ("celeba", 128, 10, 200, (500, 2000))]
TF32_TFLOPS = 495.0
HBM_TBPS = 3.35
SHAPES = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}


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


def csr_kernel_times(gen, y, a, z, R, calls=10):
    """Mean device time per call of each CSR product over dgan_loss_grad_measured_csr calls (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    gen.loss_grad_measured(y, a, z, R)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            gen.loss_grad_measured(y, a, z, R)
        torch.cuda.synchronize()
    out = {"measure": 0.0, "adjoint": 0.0}
    for ka in prof.key_averages():
        if "measured_csr_kernel" not in ka.key:           # <0>: the measurement product, <1>: the adjoint
            continue
        out["measure" if "<0>" in ka.key else "adjoint"] += ka.device_time_total / 1e3 / calls
    return out


def conv_kernel_times(gen, y, op, z, R, calls=10):
    """Mean device time per call of each convolution product over dgan_loss_grad_measured_conv calls (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    gen.loss_grad_measured(y, op, z, R)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            gen.loss_grad_measured(y, op, z, R)
        torch.cuda.synchronize()
    out = {"measure": 0.0, "adjoint": 0.0}
    for ka in prof.key_averages():
        if "measured_conv_adjoint_kernel" in ka.key:
            out["adjoint"] += ka.device_time_total / 1e3 / calls
        elif "measured_conv_kernel" in ka.key:
            out["measure"] += ka.device_time_total / 1e3 / calls
    return out


def motion_kernels(B, size=9, seed=0):
    """B random motion-blur kernels: a random walk of 2 size steps from the centre, its visits counted and normalised."""
    rs = np.random.RandomState(seed)
    ks = np.zeros((B, size, size), dtype=np.float64)
    for b in range(B):
        i = j = size // 2
        for _ in range(2 * size):
            ks[b, i, j] += 1.0
            di, dj = rs.randint(-1, 2, size=2)
            i, j = min(size - 1, max(0, i + di)), min(size - 1, max(0, j + dj))
        ks[b] /= ks[b].sum()
    return ks.astype(np.float32)


def stream_bytes(n, m, hwc):
    """Bytes each product has to move on n latent rows: G (or r) read once, r (or dy) written once."""
    m_ld = (m + 63) // 64 * 64
    return 4 * (n * hwc + n * m_ld), 4 * (n * m_ld + n * hwc)


def csr_product_bytes(n, m, hwc, nnz):
    """Algorithmic bytes of the two CSR products of one L-step on n latent rows: G (or r) read once, r (or dy) written once,
    the staged operator (int32 row pointers, int32 columns, fp32 values) and the measurements read once."""
    m_ld = (m + 63) // 64 * 64
    measure = 4 * (n * hwc + n * m_ld + (m_ld + 1) + 2 * nnz + n // 10 * m_ld)
    adjoint = 4 * (n * m_ld + n * hwc + (hwc + 1) + 2 * nnz)
    return measure, adjoint


def sparse_main(args, dev):
    from defensegan_b200 import _native as N
    from defensegan_b200.operators import ConvOperator
    res = {"card": card(), "reps": args.reps, "warmup": args.warmup, "precision": args.precision, "results": []}
    for arch, B, R, L, subs in (("mnist", 256, 10, 200, (100, 392)), ("celeba", 128, 10, 200, (1024, 4096))):
        w = O.init_generator_weights(arch)
        x = torch.tensor(O.synthetic_images(arch, w, B)).to(dev)
        h, w_, c = SHAPES[arch]
        hwc = h * w_ * c
        z0 = torch.tensor(O.sample_z0(B * R, 128)).to(dev)
        gen = N.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], precision=args.precision,
                                device=dev)
        ops = {"block2": MO.block_average_operator(h, w_, c, 2), "blur5": SO.blur_operator(h, w_, c)}
        for m in subs:
            ops["sub%d" % m] = SO.subsample_operator(m, hwc, seed=m)
        convs = {"block2": ConvOperator.box(2), "blur5": ConvOperator.gaussian(5, 1.0), "box4": ConvOperator.box(4),
                 "motion9": ConvOperator(motion_kernels(B), stride=1, padding=4)}
        ops["box4"] = ops["motion9"] = None
        r = {"arch": arch, "images": B, "restarts": R, "steps": L, "precision": args.precision, "operators": []}
        t_plain = []
        for name, a_np in ops.items():
            conv = convs.get(name)
            if a_np is None:                         # a convolution only: plain and conv calls
                m = conv.num_measurements((h, w_, c))
                lr = 10.0 * min(1.0, 4.0 * m / hwc) if m < hwc else 10.0
                y = conv(x.reshape(B, h, w_, c).double()).float()
                calls = {"plain": lambda: gen.reconstruct(x, R, L, 10.0, z_init_val=z0),
                         "conv": lambda: gen.reconstruct_measured(y, conv, R, L, lr, z_init_val=z0)}
                times = {k: [] for k in calls}
                for i in range(args.warmup + args.reps):
                    for k, fn in calls.items():
                        t = timed(fn)
                        if i >= args.warmup:
                            times[k].append(t)
                t_plain += times["plain"]
                med = {k: float(np.median(v)) for k, v in times.items()}
                e = {"operator": name, "m": m, "plain_ms": round(med["plain"], 3)}
                e.update(conv_entry(gen, conv, y, z0, B, R, L, m, hwc, med, times, h, w_, c))
                print(json.dumps(e), flush=True)
                r["operators"].append(e)
                gen._ws = None
                torch.cuda.empty_cache()
                continue
            m = a_np.shape[0]
            lr = 10.0 * min(1.0, 4.0 * m / hwc) if m < hwc else 10.0
            dense = torch.tensor(a_np).to(dev)
            csr = dense.to_sparse_csr()
            nnz = csr.values().numel()
            y = x.reshape(B, -1) @ dense.t()
            ws_dense = int(gen.lib.dgan_workspace_bytes_measured(gen._handle, B, R, m))
            ws_csr = int(gen.lib.dgan_workspace_bytes_measured_csr(gen._handle, B, R, m, nnz))
            calls = {"plain": lambda: gen.reconstruct(x, R, L, 10.0, z_init_val=z0),
                     "csr": lambda: gen.reconstruct_measured(y, csr, R, L, lr, z_init_val=z0)}
            if conv is not None:
                calls["conv"] = lambda: gen.reconstruct_measured(y, conv, R, L, lr, z_init_val=z0)
            dense_note = None
            try:
                gen.reconstruct_measured(y, dense, R, 1, lr, z_init_val=z0)
                torch.cuda.synchronize()
                calls["dense"] = lambda: gen.reconstruct_measured(y, dense, R, L, lr, z_init_val=z0)
            except (RuntimeError, torch.OutOfMemoryError) as e:
                dense_note = "not run: %s" % str(e).splitlines()[0][:200]
                gen._ws = None
                torch.cuda.empty_cache()
            times = {k: [] for k in calls}
            for i in range(args.warmup + args.reps):
                for k, fn in calls.items():
                    t = timed(fn)
                    if i >= args.warmup:
                        times[k].append(t)
            t_plain += times["plain"]
            med = {k: float(np.median(v)) for k, v in times.items()}
            kt = csr_kernel_times(gen, y, csr, z0, R)
            bm, ba = csr_product_bytes(B * R, m, hwc, nnz)
            e = {"operator": name, "m": m, "nnz": nnz,
                 "plain_ms": round(med["plain"], 3), "plain_images_per_s": round(B / med["plain"] * 1e3, 1),
                 "csr_ms": round(med["csr"], 3), "csr_images_per_s": round(B / med["csr"] * 1e3, 1),
                 "csr_spread_ms": [round(min(times["csr"]), 3), round(max(times["csr"]), 3)],
                 "csr_over_plain": round(med["csr"] / med["plain"], 4),
                 "csr_overhead_per_step_ms": round((med["csr"] - med["plain"]) / L, 4),
                 "csr_measure_product_ms": round(kt["measure"], 4), "csr_adjoint_product_ms": round(kt["adjoint"], 4),
                 "csr_measure_bytes": bm, "csr_adjoint_bytes": ba,
                 "csr_measure_hbm_share": round(bm / (kt["measure"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["measure"] else None,
                 "csr_adjoint_hbm_share": round(ba / (kt["adjoint"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["adjoint"] else None,
                 "workspace_bytes_dense": ws_dense, "workspace_bytes_csr": ws_csr}
            if conv is not None:
                e.update(conv_entry(gen, conv, y, z0, B, R, L, m, hwc, med, times, h, w_, c))
                e["conv_over_csr"] = round(med["conv"] / med["csr"], 4)
                sm, sa = stream_bytes(B * R, m, hwc)
                e["csr_measure_stream_share"] = round(sm / (kt["measure"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["measure"] else None
                e["csr_adjoint_stream_share"] = round(sa / (kt["adjoint"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["adjoint"] else None
            if "dense" in med:
                e.update({"dense_ms": round(med["dense"], 3), "dense_images_per_s": round(B / med["dense"] * 1e3, 1),
                          "dense_over_csr": round(med["dense"] / med["csr"], 3)})
            else:
                e["dense"] = dense_note
            print(json.dumps(e), flush=True)
            r["operators"].append(e)
            del dense, csr, calls
            gen._ws = None
            torch.cuda.empty_cache()
        r["plain_ms_all"] = [round(t, 3) for t in t_plain]
        gen.close()
        res["results"].append(r)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "measured_bench_sparse.json"), "w") as f:
        json.dump(res, f, indent=1)


def conv_entry(gen, conv, y, z0, B, R, L, m, hwc, med, times, h, w_, c):
    """The convolution call's columns of a --sparse row: its time, its products' times and their share of HBM on the
    stream byte count, and its workspace bytes."""
    from defensegan_b200 import _native as N
    kt = conv_kernel_times(gen, y, conv, z0, R)
    sm, sa = stream_bytes(B * R, m, hwc)
    kh, kw = conv.kernel_size
    op = N.dgan_conv_op(kh, kw, conv.padding[0], conv.padding[1], conv.stride)
    return {"kernel": [kh, kw], "stride": conv.stride, "padding": list(conv.padding), "per_image": conv.per_image,
            "conv_ms": round(med["conv"], 3), "conv_images_per_s": round(B / med["conv"] * 1e3, 1),
            "conv_spread_ms": [round(min(times["conv"]), 3), round(max(times["conv"]), 3)],
            "conv_over_plain": round(med["conv"] / med["plain"], 4),
            "conv_measure_product_ms": round(kt["measure"], 4), "conv_adjoint_product_ms": round(kt["adjoint"], 4),
            "stream_measure_bytes": sm, "stream_adjoint_bytes": sa,
            "conv_measure_hbm_share": round(sm / (kt["measure"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["measure"] else None,
            "conv_adjoint_hbm_share": round(sa / (kt["adjoint"] * 1e-3) / (HBM_TBPS * 1e12), 4) if kt["adjoint"] else None,
            "workspace_bytes_conv": int(gen.lib.dgan_workspace_bytes_measured_conv(gen._handle, B, R, ctypes.byref(op),
                                                                                    None, 0, 0))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    ap.add_argument("--user-steps", type=int, default=10)
    ap.add_argument("--sparse", action="store_true", help="compare plain, dense and CSR calls on sparse operators")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("measured_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    if args.sparse:
        return sparse_main(args, dev)
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
