"""The GPU tests' shared helpers: a handle on random weights, bit-exact comparisons, the synthetic images and z0 the
tests project, the fixture that hands back cached memory, and the one reader of the library's workspace layouts.  Import
`release_cached_memory` into a test module to use it as that module's fixture."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import defensegan_oracle as O

HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
# (arch, latent, net_dim, use_bn) of the per-layer tests, and their row counts
MATRIX = [("mnist", 128, 64, False), ("mnist", 128, 64, True), ("mnist", 100, 32, False), ("mnist", 128, 128, False),
          ("celeba", 128, 64, False), ("celeba", 200, 48, False), ("celeba", 64, 128, True)]
ROWS = [1, 300, 2560]
# tolerances of the measured projection against fp64
TOL = {"fp32": dict(fwd=2e-5, grad_rel=2e-4, grad_cos=0.999999, loss=1e-6),
       "fp16": dict(fwd=5e-3, grad_rel=6e-2, grad_cos=0.998, loss=1e-4)}


@pytest.fixture(scope="module", autouse=True)
def release_cached_memory():
    """The library allocates with cudaMalloc, outside torch's caching allocator: hand back the blocks this module left
    cached, so that the handles of later tests find the memory."""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def gen(arch, precision, use_bn=False, latent=128, net_dim=64):
    """(weights, NativeGenerator) on random weights with random biases."""
    from defensegan_b200 import _native
    dev = torch.device("cuda", 0)
    w = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, use_bn=use_bn, random_bias=True)
    g = _native.NativeGenerator(arch, [torch.as_tensor(v).to(dev) for v in w.values()], latent_dim=latent,
                                net_dim=net_dim, use_bn=use_bn, precision=precision, device=dev)
    return w, g


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    return all(torch.equal(bits(p), bits(q)) for p, q in zip(a, b))


def images(arch, w, B, seed=2):
    return torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=seed)).cuda()


def z0(n, latent=128, seed=3):
    return torch.tensor(O.sample_z0(n, latent, seed=seed)).cuda()


def rec(gen, x, R, L, lr, z0, **kw):
    return [t.clone() for t in gen.reconstruct(x, R, L, lr, z_init_val=z0, return_aux=True, **kw)]


def rec_m(gen, y, a, R, L, lr, z0, **kw):
    return [t.clone() for t in gen.reconstruct_measured(y, a, R, L, lr, z_init_val=z0, return_aux=True, **kw)]


# ---- the workspace ----

def _layout_argtypes():
    """The arguments of each dgan_debug_workspace_layout* printer between the handle and (char* buf, int len)."""
    from defensegan_b200 import _native
    i, pp = ctypes.c_int, ctypes.POINTER(_native.dgan_prune_point)
    return {"": [i],                                              # n_rows
            "_weighted": [i],                                     # n_rows
            "_measured": [i, i],                                  # n_rows, m
            "_measured_csr": [i, i, i],                           # n_rows, m, nnz
            "_measured_conv": [i, ctypes.POINTER(_native.dgan_conv_op)],   # n_rows, op
            "_pruned": [i, i, pp, i, i],                          # batch, rec_rr, sched, n_points, weighted
            "_measured_pruned": [i, i, i, i, pp, i],              # batch, rec_rr, m, nnz, sched, n_points
            "_adam": [i, i, i, i, i, pp, i],                      # batch, rec_rr, weighted, m, nnz, sched, n_points
            # batch, rec_rr, weighted, m, nnz, op, adam, sched, n_points
            "_sparse_dev": [i, i, i, i, i, ctypes.c_void_p, i, pp, i]}


DTYPES = {"f32": torch.float32, "f16": torch.float16, "i32": torch.int32, "u32": torch.int32, "u64": torch.int64}


def layout(gen, kind, *args):
    """Call dgan_debug_workspace_layout<kind> for gen's handle with args; a list of (iter, keep) pairs is passed as a
    dgan_prune_point array (NULL when empty).  Returns ({k: {off, n_rows, n_pad, bufs, meta}}, the text).  bufs maps a
    buffer's name to (type, offset in its region, dims); meta holds every other line's fields.  k is the region of a
    pruned workspace, "operator" its operator block, and 0 with offset 0 an unpruned workspace."""
    from defensegan_b200 import _native
    fn = getattr(gen.lib, "dgan_debug_workspace_layout" + kind)
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] + _layout_argtypes()[kind] + [ctypes.c_char_p, ctypes.c_int]
    args = [((_native.dgan_prune_point * len(a))(*[_native.dgan_prune_point(*p) for p in a]) if a else None)
            if isinstance(a, list) else a for a in args]
    buf = ctypes.create_string_buffer(1 << 18)
    assert fn(gen._handle, *args, buf, len(buf)) > 0, gen.lib.dgan_last_error()
    text = buf.value.decode()
    regions, cur = {}, None
    for line in text.splitlines():
        f = line.split()
        if f[0] == "region":
            cur = regions[int(f[1])] = {"off": int(f[2]), "n_rows": int(f[3]), "bufs": {}, "meta": {}}
            continue
        if f[0] == "operator":
            cur = regions["operator"] = {"off": int(f[1]), "n_rows": int(f[2]), "bufs": {}, "meta": {}}
            continue
        if cur is None:
            cur = regions[0] = {"off": 0, "bufs": {}, "meta": {}}
        if len(f) >= 3 and f[1] in DTYPES:
            cur["bufs"][f[0]] = (f[1], int(f[2]), [int(v) for v in f[3:]])
        else:
            cur["meta"][f[0]] = f[1:]
            if f[0] == "n_pad":
                cur["n_pad"] = int(f[1])
    return regions, text


def ws_base(t):
    """The address the library uses for a workspace tensor t: its first 1024-byte boundary."""
    return (t.data_ptr() + 1023) // 1024 * 1024


def view(gen, region, name):
    """Buffer `name` of a region of gen's workspace, as a tensor viewing it."""
    typ, off, dims = region["bufs"][name]
    dt = DTYPES[typ]
    start = ws_base(gen._ws) - gen._ws.data_ptr() + region["off"] + off
    return gen._ws[start:start + int(np.prod(dims)) * dt.itemsize].view(dt).view(*dims)


def views(gen, region):
    return {name: view(gen, region, name) for name in region["bufs"]}


def read(gen, region, name):
    """A copy of buffer `name` of a region, after the stream's work."""
    torch.cuda.synchronize()
    return view(gen, region, name).clone()


def read_call(native, w, arch, latent, net_dim, use_bn, precision, n_rows):
    """The workspace a call for n_rows rows left, by name, and the reference network at the handle's padded widths."""
    import layer_ref as R
    ws = layout(native, "", n_rows)[0][0]
    assert ws["meta"]["n_rows"] == [str(n_rows)]
    net = R.Net(arch, latent, net_dim, use_bn, precision, [int(v) for v in ws["meta"]["widths"]], w,
                torch.device("cuda", 0))
    return views(native, ws), net


def check_products(ws, n, rec_rr, m, hwc, precision):
    """r = A G - y and dy = (2/m) A^T r of the last measured call on n latent rows (rec_rr restarts per image) against
    fp64 on the operands the kernels read (the measured workspace's buffers), each within the bound of its arithmetic
    (test_each_measurement_product_on_its_stored_operands); the padded measurements of r exact zeros.  Returns the
    largest error over its bound of r and of dy."""
    u = 2.0 ** -24
    rnd = 2.0 ** -10 if precision == "fp16" else 0.0      # two operands rounded to TF32, 2^-11 each
    m_ld = ws["am"].shape[0]

    def bound(x, wt, k):
        g = k * u / (1 - k * u)
        return (rnd + g) * (x.abs().double() @ wt.abs().double().t())

    g = ws["y"][:n]
    y_rows = ws["ym"][:n // rec_rr].repeat_interleave(rec_rr, dim=0)
    r64 = g.double() @ ws["am"].double().t() - y_rows.double()
    r = ws["r"][:n]
    err = (r.double() - r64).abs()
    lim = bound(g, ws["am"], hwc) + u * r64.abs() + 1e-30
    r_ratio = float((err / lim).max())
    assert bool((err <= lim).all()), "measurement product (r): max err / bound %.3g" % r_ratio
    assert not r[:, m:].any()                              # padded measurements are exact zeros
    dy64 = (2.0 / m) * (r.double() @ ws["amt"].double().t())
    dy = ws["dym"][:n]
    err = (dy.double() - dy64).abs()
    lim = (2.0 / m) * bound(r, ws["amt"], m_ld) * (1 + 2 * u) + 2 * u * dy64.abs() + 1e-30
    dy_ratio = float((err / lim).max())
    assert bool((err <= lim).all()), "adjoint product (dy): max err / bound %.3g" % dy_ratio
    return r_ratio, dy_ratio


def gsum(g):
    """The partial sums g[0] + g[1] + ... in the order the library adds them."""
    gs = g[0].clone()
    for p in range(1, g.shape[0]):
        gs = gs + g[p]
    return gs


def option_layout(gen, batch, R, weighted=0, m=0, nnz=-1, sched=None, adam=True):
    """(region 0, text) of the printer a call with these options plans: the Adam printer, else the pruned, measured
    [CSR], weighted or plain one."""
    if adam:
        regions, text = layout(gen, "_adam", batch, R, weighted, m, nnz, list(sched or []), len(sched or []))
    elif sched:
        regions, text = layout(gen, "_pruned", batch, R, list(sched), len(sched), weighted)
    elif m > 0:
        regions, text = (layout(gen, "_measured_csr", batch * R, m, nnz) if nnz >= 0
                         else layout(gen, "_measured", batch * R, m))
    else:
        regions, text = layout(gen, "_weighted" if weighted else "", batch * R)
    return regions[0], text


def option_lr(kw):
    """The step of a projection with options kw: Adam's or momentum's."""
    return 0.02 if "adam" in kw else 0.5
