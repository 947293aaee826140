"""Developer aid (no GPU needed): print the planner's numbers for every tensor-core layer-direction.
Usage: python tools/plan_stats.py [mnist|celeba] [batch] [R] [CTA pairs] [library] [--slots DIR=MAXB] [--window DIR=WH,WW,SY,SX]
--slots plans layer-direction DIR (the row index of the table, from 0) with exactly MAXB accumulator slots per round;
--window plans it on exactly the window WH x WW with strides (SY, SX), e.g. to compare two builds at the same window."""
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
window = None
if "--window" in sys.argv:
    i = sys.argv.index("--window")
    d, shape = sys.argv[i + 1].split("=")
    force_dir, window = int(d), [int(v) for v in shape.split(",")]
    del sys.argv[i:i + 2]
dataset = sys.argv[1] if len(sys.argv) > 1 else "mnist"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 256
R = int(sys.argv[3]) if len(sys.argv) > 3 else 10
pairs = int(sys.argv[4]) if len(sys.argv) > 4 else 74
lib = ctypes.CDLL(sys.argv[5]) if len(sys.argv) > 5 else ctypes.CDLL(_native.build_library())
desc = _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[dataset], 128, 64, 0, _native.PRECISIONS["fp16"])
buf = ctypes.create_string_buffer(1 << 16)
lib.dgan_debug_plan_stats_slots.restype = ctypes.c_int
lib.dgan_debug_plan_stats_slots.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_char_p, ctypes.c_int]
if window is None:
    n = lib.dgan_debug_plan_stats_slots(ctypes.byref(desc), batch * R, pairs, force_dir, force_maxb, buf, len(buf))
else:
    lib.dgan_debug_plan_stats_window.restype = ctypes.c_int
    n = lib.dgan_debug_plan_stats_window(ctypes.byref(desc), batch * R, pairs, force_dir, force_maxb, *window, buf, len(buf))
assert n > 0
print(buf.value.decode())
