"""Developer aid (no GPU needed): print the planner's numbers for every tensor-core layer-direction.
Usage: python tools/plan_stats.py [mnist|celeba] [batch] [R] [CTA pairs] [library] [--slots DIR=MAXB] [--window DIR=WH,WW,SY,SX]
                                 [--latent_dim N] [--net_dim N] [--use_bn]
--latent_dim / --net_dim / --use_bn plan that generator (default 128 / 64 / no BN); the handle pads each width (see
DESIGN.md section 2), and the next two columns show the share of each direction's k16 MMAs that multiply real channels
and its steps per CTA pair (what each consumer warp pays a fixed per-step cost for).  The MMA columns of the table count
every slot of every round, as the planner's time model does; the last three (default plans only, no --slots or --window)
give what the kernel issues: the k16 MMAs issued, the zero-tile k16 MMAs it skips (rounds with 2 or 4 slots and
64-channel ops issue only their real ops) and the busiest pair's estimated tensor time for the MMAs issued;
--slots plans layer-direction DIR (the row index of the table, from 0) with exactly MAXB accumulator slots per round;
--window plans it on exactly the window WH x WW with strides (SY, SX), e.g. to compare two builds at the same window.
A second table (default plans only) gives the item order of each plan (lpt, or band+ / band- with the direction the
bands are walked in), its row pairs per band, the busiest pair's cost-model load under LPT and under that order, the
bytes staged as activation tiles and as weight tiles, the unique input (the distinct activation tiles read) and the
working set: the peak, over the cost model's timeline of every pair, of the bytes of activation tiles between their first
and last load.  Set against the 50 MB L2, it shows without a GPU which directions the order can help; --order lpt gives
the table for the LPT order."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from defensegan_b200 import _native

force_dir, force_maxb = -1, 0
if "--slots" in sys.argv:
    i = sys.argv.index("--slots")
    force_dir, force_maxb = (int(v) for v in sys.argv[i + 1].split("="))
    del sys.argv[i:i + 2]
widths = {"--latent_dim": 128, "--net_dim": 64}
for flag in widths:
    if flag in sys.argv:
        i = sys.argv.index(flag)
        widths[flag] = int(sys.argv[i + 1])
        del sys.argv[i:i + 2]
use_bn = "--use_bn" in sys.argv
if use_bn:
    sys.argv.remove("--use_bn")
window = None
if "--window" in sys.argv:
    i = sys.argv.index("--window")
    d, shape = sys.argv[i + 1].split("=")
    force_dir, window = int(d), [int(v) for v in shape.split(",")]
    del sys.argv[i:i + 2]
order = 1
if "--order" in sys.argv:
    i = sys.argv.index("--order")
    order = {"lpt": 0, "band": 1}[sys.argv[i + 1]]
    del sys.argv[i:i + 2]
dataset = sys.argv[1] if len(sys.argv) > 1 else "mnist"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 256
R = int(sys.argv[3]) if len(sys.argv) > 3 else 10
pairs = int(sys.argv[4]) if len(sys.argv) > 4 else 74
lib = ctypes.CDLL(sys.argv[5]) if len(sys.argv) > 5 else ctypes.CDLL(_native.build_library())
latent, nd = widths["--latent_dim"], widths["--net_dim"]
desc = _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[dataset], latent, nd, int(use_bn), _native.PRECISIONS["fp16"])
buf = ctypes.create_string_buffer(1 << 16)
lib.dgan_debug_plan_stats_slots.restype = ctypes.c_int
lib.dgan_debug_plan_stats_slots.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_char_p, ctypes.c_int]
if window is None:
    n = lib.dgan_debug_plan_stats_slots(ctypes.byref(desc), batch * R, pairs, force_dir, force_maxb, buf, len(buf))
else:
    lib.dgan_debug_plan_stats_window.restype = ctypes.c_int
    n = lib.dgan_debug_plan_stats_window(ctypes.byref(desc), batch * R, pairs, force_dir, force_maxb, *window, buf, len(buf))
if n <= 0:
    lib.dgan_last_error.restype = ctypes.c_char_p
    raise SystemExit((lib.dgan_last_error() or b"planning failed").decode())
# real (unpadded) N and K of each layer-direction; a column block "name[a:b]" has the real channels of [a, b)
img = 48 if dataset == "celeba" else 16
real = {"Linear.fwd": (4 * nd, latent), "Linear.bwd": (latent, 4 * nd), "Generator.2.fwd": (2 * nd, 4 * nd),
        "Generator.2.bwd": (4 * nd, 2 * nd), "Generator.3.fwd": (nd, 2 * nd), "Generator.3.bwd": (2 * nd, nd),
        "Generator.5.fwd": (nd, nd), "Generator.5.bwd": (nd, nd), "last.fwd": (img, nd), "last.bwd": (nd, img)}
lines = buf.value.decode().strip().splitlines()
issue = {}
if window is None and force_dir < 0:
    ibuf = ctypes.create_string_buffer(1 << 16)
    lib.dgan_debug_plan_issue_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_issue_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    if lib.dgan_debug_plan_issue_stats(ctypes.byref(desc), batch * R, pairs, ibuf, len(ibuf)) > 0:
        for row in ibuf.value.decode().strip().splitlines()[1:]:
            col = row.split(" | ")
            issue[col[0]] = " | ".join(col[2:])
out = [lines[0] + " | real k16 MMAs (share) | steps per CTA pair" +
       (" | k16 MMAs issued | zero-tile k16 MMAs skipped | busiest pair: est. tensor us, issued" if issue else "")]
for line in lines[1:-1]:
    col = line.split(" | ")
    name, n, k = col[0], int(col[1]), int(col[2])
    rn, rk = real[name.split("[")[0]]
    if "[" in name:
        a, b = (int(v) for v in name[name.index("[") + 1:-1].split(":"))
        rn = max(0, min(b, rn) - a)
    share = min(rn, n) * min(rk, k) / (n * k)
    out.append(line + " | %d (%.2f) | %.1f" % (round(int(col[14]) * share), share, int(col[6]) / pairs) +
               (" | " + issue[name] if name in issue else ""))
out.append(lines[-1])
print("\n".join(out))
if window is None and force_dir < 0:
    obuf = ctypes.create_string_buffer(1 << 16)
    lib.dgan_debug_plan_order_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_order_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_char_p, ctypes.c_int]
    if lib.dgan_debug_plan_order_stats(ctypes.byref(desc), batch * R, pairs, order, obuf, len(obuf)) > 0:
        print()
        print(obuf.value.decode().strip())
