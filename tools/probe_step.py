"""Developer aid, needs a library built with -DDGAN_PROBE (DGAN_LIB=...): per tensor-core kernel instantiation, the
distribution over CTAs of the cycles from the PDL wait to the end of the CTA's work (mean over the launches of one
projection): a wide distribution = the static item assignment leaves SMs idle at the kernel boundary.
The second table splits the first consumer warp's cycles into the operand wait, MMA issue, the wgmma_wait1 after each
round, the wgmma_wait0 at the end of each item and the epilogues, as shares of its busy cycles, and what is left ("rest")
into the record wait (operands landed -> the step's MMA record read and first used), the item head (end of an epilogue
-> the next item's first operand wait), the end wait (last epilogue -> every warp of the CTA done) and the remainder;
with the steps per CTA and launch, and the record wait in cycles per step.  The epilogue's share is split further into
waiting for its global inputs (mask words, bias, image and weight pairs), waiting for a staging buffer of the TMA store,
and the rest of it; in the TMA-store epilogues that rest splits into the register work of each 64-column unit (bias, ReLU
or mask, fp16 conversion, the ReLU mask words), writing its staging buffer, and the fence.proxy.async before its store.
Usage: DGAN_LIB=build_ab/probe.so python tools/probe_step.py [mnist|celeba] [batch] [L] [--json]
(--json: one JSON object with the time-ordered busy / hand-over table instead of the text tables; bench.py uses it)"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from defensegan_b200.models.gan import dataset_gan_dict

as_json = "--json" in sys.argv
argv = [a for a in sys.argv if a != "--json"]
dataset = argv[1] if len(argv) > 1 else "mnist"
B = int(argv[2]) if len(argv) > 2 else 256
L = int(argv[3]) if len(argv) > 3 else 50
if as_json:
    _stdout, sys.stdout = sys.stdout, sys.stderr       # the text tables go to stderr, the JSON object alone to stdout
gan = dataset_gan_dict[dataset](test_mode=True, verbose=False, precision="fp16", batch_size=50)
gan.rec_rr, gan.rec_iters = 10, L
g = torch.Generator().manual_seed(0)
x = torch.rand(B, *gan.image_dim, generator=g).cuda()
z0 = (torch.randn(B * 10, 128, generator=g) * 128 ** -0.5).cuda()
lib = gan._native.lib if hasattr(gan, "_native") and gan._native is not None else None
gan.reconstruct(x, z_init_val=z0)
torch.cuda.synchronize()
lib = gan._native.lib
W = 21                                              # counters per CTA (TC2_PROBE_WORDS)
buf = (ctypes.c_ulonglong * (48 * 160 * W))()
lib.dgan_debug_probe_read.restype = ctypes.c_int
lib.dgan_debug_probe_read.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
assert lib.dgan_debug_probe_read(buf) == 0          # discard the first call (schedule upload, graph capture)
gan.reconstruct(x, z_init_val=z0)
torch.cuda.synchronize()
assert lib.dgan_debug_probe_read(buf) == 0
a = np.frombuffer(buf, dtype=np.uint64).reshape(48, 160, W).astype(np.float64)
# algorithmic MACs per launch of the MNIST kernels (in-bounds pairs x C_in x C_out x rows), for the busy-time TFLOP/s column
rows = B * 10
kind_flops, layer_names = {}, {}
if dataset != "celeba":
    layer_names = {(256, "bias+relu"): "Linear.fwd", (128, "float-out"): "Linear.bwd", (128, "bias+relu"): "Generator.2.fwd",
                   (256, "mask"): "Generator.2.bwd", (64, "bias+relu"): "Generator.3.fwd", (128, "mask"): "Generator.3.bwd",
                   (16, "final-sigmoid"): "Generator.5+loss.fwd", (64, "mask"): "Generator.5.bwd"}
    kind_flops = {(256, "bias+relu"): 524288.0 * rows, (128, "float-out"): 524288.0 * rows, (128, "bias+relu"): 7372800.0 * rows,
                  (256, "mask"): 7372800.0 * rows, (64, "bias+relu"): 8388608.0 * rows, (128, "mask"): 8388608.0 * rows,
                  (16, "final-sigmoid"): 287296.0 * rows, (64, "mask"): 287296.0 * rows}
NT = [256, 128, 64, 48, 16]
EP = ["bias+relu", "bias", "mask", "none", "final-sigmoid", "final-tanh", "float-out", "?"]
# keys 40 - 43: the Huber final kinds (tc2_probe_key)
HUBER = [(16, "final-sigmoid-huber"), (48, "final-tanh-huber"), (16, "final-sigmoid-huber-w"), (48, "final-tanh-huber-w")]


def kind(k):
    return HUBER[k - 40] if k >= 40 else (NT[k // 8], EP[k % 8])


raw = np.frombuffer(buf, dtype=np.uint64).reshape(48, 160, W)
print("kernel <N, epilogue> | launches | cycles from PDL wait to CTA end: mean / min / max over CTAs | (max-mean)/max | trigger->wait mean | MMA operand wait mean (leaders) | set-up cycles mean | last launch, ns from its first CTA entry: last entry / first operands (mean, leaders) / first CTA end / last CTA end")
timeline, split = [], {}
for k in range(48):
    cnt = a[k, :, 1]
    act = cnt > 0
    if not act.any():
        continue
    dur = a[k, act, 0] / cnt[act]
    pre = a[k, act, 2] / cnt[act]
    wf = a[k, act, 3] / cnt[act]
    lead = wf > 0
    setup = a[k, act, 4] / cnt[act]
    g0 = raw[k, act, 5].astype(np.int64); g1 = raw[k, act, 6].astype(np.int64); gf = raw[k, act, 7].astype(np.int64)
    t0 = g0.min()
    print("<%d, %s> | %d | %.0f / %.0f / %.0f | %.3f | %.0f | %.0f | %.0f | %d / %.0f / %d / %d   [abs first entry %d, last end %d]" % (
        *kind(k), int(cnt[act].max()), dur.mean(), dur.min(), dur.max(), (dur.max() - dur.mean()) / dur.max(), pre.mean(),
        wf[lead].mean() if lead.any() else 0, setup.mean(), g0.max() - t0, (gf[gf > 0] - t0).mean() if (gf > 0).any() else -1, g1.min() - t0, g1.max() - t0, t0, g1.max()))
    # the first consumer warp of each CTA (thread 0): shares of its busy cycles, means over CTAs
    sh = [float((a[k, act, c] / a[k, act, 0]).mean()) for c in (3, 8, 9, 10, 11, 12, 13, 14)]
    steps = a[k, act, 15]
    sh += [float((steps / cnt[act]).mean()), float((a[k, act, 12][steps > 0] / steps[steps > 0]).mean()) if (steps > 0).any() else 0.0]
    sh += [float((a[k, act, c] / a[k, act, 0]).mean()) for c in (16, 17, 18, 19, 20)]
    split[layer_names.get(kind(k), "<%d, %s>" % kind(k))] = dict(
        zip(("operand_wait", "issue", "wgmma_wait1", "wgmma_wait0", "epilogue", "record_wait", "item_head", "end_wait",
             "steps_per_cta", "record_wait_cycles_per_step", "epilogue_input_wait", "epilogue_staging_wait",
             "epilogue_registers", "epilogue_staging_stores", "epilogue_fence"),
            [round(v, 3) for v in sh]))
    timeline.append((int(t0), layer_names.get(kind(k), "<%d, %s>" % kind(k)), int(g0.max()), float(gf[gf > 0].mean()) if (gf > 0).any() else float(g0.max()),
                     int(g1.max()), 2.0 * kind_flops.get(kind(k), 0.0)))
# the last launches of the kernels, in time order: how long each was busy and what the hand-over from its predecessor cost
timeline.sort()
print()
print("last L-step, in time order | busy us (last CTA entry -> last CTA end) | hand-over us (predecessor's last CTA end -> first operands landed) | algorithmic TFLOP/s while busy")
prev_end = None
tot_busy = tot_gap = 0.0
for t0, name, last_entry, first_full, last_end, flops in timeline:
    busy = (last_end - last_entry) / 1e3
    gap = (first_full - prev_end) / 1e3 if prev_end is not None and abs(first_full - prev_end) < 1e5 else float("nan")
    print("%s | %.1f | %.1f | %s" % (name, busy, gap, ("%.0f" % (flops / busy / 1e6)) if flops else "-"))
    tot_busy += busy
    if gap == gap:
        tot_gap += gap
    prev_end = last_end
print("sum | %.1f | %.1f |" % (tot_busy, tot_gap))
print()
print("first consumer warp, share of its busy cycles | operand wait | MMA issue | wgmma_wait1 | wgmma_wait0 | epilogue | rest"
      " | of rest: record wait | item head | end wait | remainder | steps per CTA | record wait, cycles per step"
      " | of epilogue: input wait | staging wait | rest | of rest (TMA-store epilogues): register work | staging stores"
      " | fence | remainder")
for name, d in split.items():
    v = list(d.values())
    rest = 1.0 - sum(v[:5])
    e_rest = v[4] - v[10] - v[11]
    print("%s | %s | %.3f | %s | %.3f | %.1f | %.0f | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f" % (
        name, " | ".join("%.3f" % x for x in v[:5]), rest, " | ".join("%.3f" % x for x in v[5:8]), rest - sum(v[5:8]), v[8], v[9],
        v[10], v[11], e_rest, v[12], v[13], v[14], e_rest - sum(v[12:15])))
if as_json:
    import json
    rows_out, prev_end = [], None
    for t0, name, last_entry, first_full, last_end, flops in timeline:
        busy = (last_end - last_entry) / 1e3
        gap = (first_full - prev_end) / 1e3 if prev_end is not None and abs(first_full - prev_end) < 1e5 else None
        rows_out.append({"kernel": name, "busy_us": round(busy, 2), "handover_us": None if gap is None else round(gap, 2),
                         "tflops_while_busy": round(flops / busy / 1e6, 1) if flops else None, "consumer_share": split.get(name)})
        prev_end = last_end
    sys.stdout = _stdout
    print(json.dumps({"dataset": dataset, "batch": B, "rec_rr": 10, "rec_iters": L, "kernels": rows_out,
                      "sum_busy_us": round(tot_busy, 1), "sum_handover_us": round(tot_gap, 1),
                      "how": "last L-step of one call; per CTA %globaltimer stamps at kernel entry, first operands landed, end of work "
                             "(library built with -DDGAN_PROBE); busy = last CTA entry -> last CTA end, hand-over = predecessor's last "
                             "CTA end -> first operands landed"}))
