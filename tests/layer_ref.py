"""fp64 references of each layer-direction of the generator, on the operands a kernel actually read, and the per-element
bound a kernel's output must meet.  Shared by test_gpu_layers.py (the buffers a call leaves in the workspace) and
test_host_layers.py (a CPU emulation, and the same emulation with seeded defects, which the bound must reject).

A layer-direction is checked on its own stored input (fp16 on the tensor-core path, fp32 on the CUDA-core path) and the
caller's weights rounded as the handle rounds them (fp16 RN on the tensor-core path), so no ReLU-mask flip carries in
from an earlier layer.  What is left is the kernel's fp32 accumulation order and its output rounding:

    |got - ref| <= 1/2 ulp(out type) + gamma * sum |a| |w|     (sum |a||w|: the same op on |a| and |w|, plus |bias|)

  tensor cores:  gamma = (k16 MMAs per output + 1) * 2^-22  (one fp32 rounding per k16 MMA, with a factor 2 of margin)
  CUDA cores:    gamma = (FMAs per output + 1) * 2^-24      (sequential fp32 FMAs; 1/2 ulp of an fp32 output included)

Storage layouts (carve() in csrc/dgan_api.cu, read through dgan_debug_workspace_layout): activations and gradients are
[pixel][n_pad][channel], pixel = row * raster + col; ReLU mask bit j of word [(q * n_pad + n) * (C / 64) + g] is set iff
the fp32 output at channel g * 64 + j is > 0 (TcFinalArgs); the last layer's d(pre) on the tensor-core path is the block
tensor [n_blocks][n_pad][16 * C] with pixel (4 by + li, 4 bx + lj) in block by * (w / 4) + bx at column
(li * 4 + lj) * C + c (block_index in kernels_vjp.cuh)."""
from __future__ import annotations

import functools

import torch

from oracle import defensegan_oracle as O

GRAD_SCALE = 64.0        # the tensor-core path's fixed d(pre) scale (TcState::grad_scale)
LINEAR_SPLIT = 4         # partial sums of the tensor-core Linear backward (TC_LINEAR_SPLIT), 4 pixels each
# absolute error of y = act(pre) from the activation's fast-math exp and divide (tensor-core epilogue) or expf / tanhf
ACT_EPS = {"fp16": 2.0 ** -18, "fp32": 2.0 ** -21}


# ------------------------------------------------------------------------------------------------------------------
# the network: layer-directions, their geometry and weights
# ------------------------------------------------------------------------------------------------------------------
class Net:
    """Geometry of one handle: GEMM layers 0 (the Linear) .. nl-1 and the last layer, at real and padded widths."""

    def __init__(self, arch, latent, net_dim, use_bn, precision, padded, weights, device):
        self.arch, self.latent, self.net_dim, self.use_bn, self.precision = arch, latent, net_dim, use_bn, precision
        self.celeba = arch == "celeba"
        self.c_img = 3 if self.celeba else 1
        lat_p, c4p, c2p, c1p = padded
        nd = net_dim
        # (name, c_in, c_out, c_in padded, c_out padded, h_in, h_used, in_raster, relu, bn)
        if self.celeba:
            sp = [("Generator.2", 4 * nd, 2 * nd, c4p, c2p, 4, 8, 4, True, use_bn),
                  ("Generator.3", 2 * nd, nd, c2p, c1p, 8, 16, 8, True, use_bn),
                  ("Generator.5", nd, nd, c1p, c1p, 16, 32, 16, False, False)]
        elif use_bn:
            sp = [("Generator.2", 4 * nd, 2 * nd, c4p, c2p, 4, 8, 4, True, True),
                  ("Generator.3", 2 * nd, nd, c2p, c1p, 7, 14, 8, True, True)]
        else:
            sp = [("Generator.2", 4 * nd, 2 * nd, c4p, c2p, 4, 7, 4, True, False),
                  ("Generator.3", 2 * nd, nd, c2p, c1p, 7, 14, 7, True, False)]
        self.layers = [dict(name="Linear", c_in=latent, c_out=4 * nd, c_in_p=lat_p, c_out_p=c4p, h_used=4, raster_out=4,
                            relu=True, bn=use_bn, p_in=1)]
        for (nm, ci, co, cip, cop, h_in, h_used, raster, relu, bn) in sp:
            self.layers.append(dict(name=nm, c_in=ci, c_out=co, c_in_p=cip, c_out_p=cop, h_in=h_in, h_used=h_used,
                                    in_raster=raster, raster_out=h_used, relu=relu, bn=bn))
        self.nl = len(self.layers)
        self.fh = sp[-1][6]                       # the last layer's input side (14 or 32); the image is 2 * fh
        self.last_name = "Generator.6" if self.celeba else "Generator.5"
        self.act = "tanh" if self.celeba else "sigmoid"
        rnd = (lambda t: t.half().double()) if precision == "fp16" else (lambda t: t.double())
        W = {k: torch.as_tensor(v).to(device) for k, v in weights.items()}
        self.w, self.b, self.bn = [], [], []
        self.w.append(rnd(W["Generator.Input/Generator.Input.W"]))
        self.b.append(W["Generator.Input/Generator.Input.b"].double())
        names = [l["name"] for l in self.layers[1:]] + [self.last_name]
        for nm in names:
            self.w.append(rnd(W["%s/%s.Filters" % (nm, nm)]))
            self.b.append(W["%s/%s.Biases" % (nm, nm)].double())
        for i in range(1, 4):
            if use_bn:
                self.bn.append((W["Generator.BN%d.offset" % i].double().reshape(-1), W["Generator.BN%d.scale" % i].double().reshape(-1)))

    def pairs(self, l, direction):
        """Products (pairs of an input pixel and a weight tile) summed into one output of layer-direction (l, direction),
        from the geometry: l = nl is the last layer (tensor cores: its 4x4 output blocks are the GEMM's pixels)."""
        if l == 0:
            return 1 if direction == "fwd" else 16 // (LINEAR_SPLIT if self.precision == "fp16" else 1)
        if l == self.nl:
            fwd, bwd = deconv_pair_counts(self.fh, 2 * self.fh, 4 if self.precision == "fp16" else 1)
        else:
            L = self.layers[l]
            fwd, bwd = deconv_pair_counts(L["h_in"], L["h_used"], 1)
        return fwd if direction == "fwd" else bwd

    def k16(self, K):
        return (K + 15) // 16

    def gamma(self, pairs, K):
        """The accumulation bound's factor for outputs summing `pairs` products of K (padded) channels each."""
        if self.precision == "fp16":
            return (pairs * self.k16(K) + 1) * 2.0 ** -22
        return (pairs * K + 1) * 2.0 ** -24


@functools.lru_cache(maxsize=None)
def deconv_pair_counts(h_in, h_used, block):
    """The most (input pixel, weight tile) pairs any output of a 5x5 / stride-2 transposed conv on h_in x h_in inputs (the
    first h_used x h_used outputs kept) sums, forward and backward.  block = 1: a tile is a tap; block = 4: the outputs
    are grouped into 4x4 blocks and a tile is an (input pixel, block) pair's weights, as in the tensor-core last layer."""
    fwd, bwd = {}, {}
    for o in range(h_in):
        for p in range(h_in):
            for ka in range(5):
                for kb in range(5):
                    i, j = 2 * o + ka - 1, 2 * p + kb - 1
                    if 0 <= i < h_used and 0 <= j < h_used:
                        out = (i // block, j // block)
                        fwd.setdefault(out, set()).add((o, p) if block > 1 else (o, p, ka, kb))
                        bwd.setdefault((o, p), set()).add(out if block > 1 else (i, j, ka, kb))
    return max(len(s) for s in fwd.values()), max(len(s) for s in bwd.values())


# ------------------------------------------------------------------------------------------------------------------
# layouts
# ------------------------------------------------------------------------------------------------------------------
def to_nhwc(buf, n, raster, c):
    """[raster^2][n_pad][C] -> [n][raster][raster][c] (real rows and channels), fp64."""
    return buf[:, :n, :c].double().permute(1, 0, 2).reshape(n, raster, raster, c)


def from_nhwc(x):
    """[n][r][r][c] -> [r^2][n][c]."""
    n, r, r2, c = x.shape
    return x.reshape(n, r * r2, c).permute(1, 0, 2)


def block_perm(w_out, c, device):
    """Index of each element of an image row [w_out][w_out][c] (NHWC flat) in the block tensor's (block, column) plane:
    returns (blk, col) index tensors (block_index of kernels_vjp.cuh)."""
    r = torch.arange(w_out * w_out * c, device=device)
    pix, co = r // c, r % c
    row, col = pix // w_out, pix % w_out
    blk = (row // 4) * (w_out // 4) + col // 4
    k = ((row % 4) * 4 + col % 4) * c + co
    return blk, k


def blocks_to_nhwc(dblk, n, w_out, c):
    """[n_blocks][n_pad][16 c] -> [n][w_out][w_out][c], fp64."""
    blk, k = block_perm(w_out, c, dblk.device)
    return dblk[:, :n, :].double()[blk, :, k].t().reshape(n, w_out, w_out, c)


def unpack_mask(words, c_pad):
    """u64 words [P][n_pad][C/64] (as int64) -> bool [P][n_pad][C]."""
    sh = torch.arange(64, device=words.device, dtype=torch.int64)
    bits = (words.unsqueeze(-1) >> sh) & 1
    return bits.reshape(words.shape[0], words.shape[1], c_pad).bool()


# ------------------------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------------------------
def half_ulp(x, out_type):
    """1/2 ulp of |x| in the output type (fp16 subnormals included)."""
    if out_type == "f16":
        lo, mant = 2.0 ** -14, 10
    else:
        lo, mant = 2.0 ** -126, 23
    a = x.abs().clamp_min(lo)
    return torch.exp2(torch.floor(torch.log2(a)) - mant) * 0.5


class Stats:
    """Per layer-direction: the largest accumulation error over its bound, and the fraction of fp16 outputs equal to
    RN16(ref)."""

    def __init__(self):
        self.rows = {}

    def add(self, key, ratio, biteq):
        r, b, cnt = self.rows.get(key, (0.0, 0.0, 0))
        self.rows[key] = (max(r, ratio), b + (biteq if biteq is not None else 0.0), cnt + (1 if biteq is not None else 0))

    def lines(self):
        out = []
        for k, (r, b, c) in self.rows.items():
            out.append("%-34s max err/bound %.3f%s" % (k, r, "  bit-equal %.4f" % (b / c) if c else ""))
        return out


def check_close(name, got, ref, absref, gamma, out_type, stats, extra=None, where=None):
    """Assert |got - ref| <= 1/2 ulp + gamma * absref (+ extra) elementwise; got/ref/absref are [P][n][c] (or any shape,
    `where` naming the axes).  Records the ratio of the error beyond the output rounding to gamma * absref."""
    got = got.double()
    err = (got - ref).abs()
    hu = half_ulp(torch.maximum(ref.abs(), got.abs()), out_type) if out_type == "f16" else torch.zeros_like(ref)
    acc = gamma * absref
    if extra is not None:
        acc = acc + extra
    bound = hu + acc
    bad = err > bound
    excess = (err - hu).clamp_min(0)
    ratio = float((excess / acc.clamp_min(1e-300)).max()) if err.numel() else 0.0
    biteq = None
    if out_type == "f16" and got.numel():
        biteq = float((got == ref.half().double()).double().mean())
    stats.add(name, ratio, biteq)
    if bool(bad.any()):
        idx = [int(i) for i in torch.nonzero(bad)[0]]
        axes = where or ["pixel", "row", "channel"]
        loc = ", ".join("%s %d" % (a, i) for a, i in zip(axes, idx))
        if "channel" in axes:
            loc += ", column block %d" % (idx[axes.index("channel")] // 256)
        raise AssertionError("%s: %d elements out of bound; first at %s: got %.9g ref %.9g |err| %.3g bound %.3g "
                             "(gamma sum|a||w| %.3g)" % (name, int(bad.sum()), loc, float(got[tuple(idx)]),
                                                          float(ref[tuple(idx)]), float(err[tuple(idx)]),
                                                          float(bound[tuple(idx)]), float(acc[tuple(idx)])))


def check_mask(name, mask, pre_ref, tol):
    """ReLU mask bits [P][n][c] == [pre > 0] wherever |pre| > tol."""
    sure = pre_ref.abs() > tol
    bad = sure & (mask != (pre_ref > 0))
    if bool(bad.any()):
        idx = [int(i) for i in torch.nonzero(bad)[0]]
        raise AssertionError("%s mask: %d bits wrong; first at pixel %d, row %d, channel %d (column block %d): pre %.6g"
                             % (name, int(bad.sum()), idx[0], idx[1], idx[2], idx[2] // 256, float(pre_ref[tuple(idx)])))


def check_zero_pad(name, buf, c_real):
    """Every channel at or above the real width is exactly 0 (the width rule)."""
    tail = buf[..., c_real:]
    if tail.numel() and bool((tail != 0).any()):
        idx = [int(i) for i in torch.nonzero(tail != 0)[0]]
        raise AssertionError("%s: padded channel %d is %r at %s" % (name, c_real + idx[-1], float(tail[tuple(idx)]), idx))


# ------------------------------------------------------------------------------------------------------------------
# the references (fp64)
# ------------------------------------------------------------------------------------------------------------------
def deconv(x, f, b):
    return O.tf_deconv_same(x, f, b)


def deconv_dinput(dout, f):
    """The backward-to-input of tf_deconv_same (no bias): the vector-Jacobian product in x."""
    n, h2, w2, _ = dout.shape
    x = torch.zeros(n, h2 // 2, w2 // 2, f.shape[3], dtype=torch.float64, device=dout.device, requires_grad=True)
    with torch.enable_grad():
        (g,) = torch.autograd.grad(O.tf_deconv_same(x, f, None), x, dout)
    return g


def linear_fwd_ref(net, z_in, n, bias=True):
    """Linear on the stored input [1][n_pad][latent]: -> pre [16][n][c4], sum |a||w| [16][n][c4]."""
    L = net.layers[0]
    a = z_in[0, :n, :L["c_in"]].double() if z_in.dim() == 3 else z_in[:n, :L["c_in"]].double()
    W, b = net.w[0], net.b[0]
    pre = a @ W
    ab = a.abs() @ W.abs()
    if bias:
        pre = pre + b
        ab = ab + b.abs()
    c = L["c_out"]
    return pre.reshape(n, 16, c).permute(1, 0, 2), ab.reshape(n, 16, c).permute(1, 0, 2)


def deconv_fwd_ref(net, l, x_store, n, bias=True):
    """Generator layer l (>= 1) on its stored input [raster^2][n_pad][C_in]: -> pre [h_used^2][n][c_out], sum |a||w|."""
    L = net.layers[l]
    x = to_nhwc(x_store, n, L["in_raster"], L["c_in"])[:, :L["h_in"], :L["h_in"], :]
    f, b = net.w[l], net.b[l]
    hu = L["h_used"]
    pre = deconv(x, f, b if bias else None)[:, :hu, :hu, :]
    ab = deconv(x.abs(), f.abs(), b.abs() if bias else None)[:, :hu, :hu, :]
    return from_nhwc(pre), from_nhwc(ab)


def deconv_bwd_ref(net, l, dout_store, n):
    """Backward of layer l (>= 1) into its input, from the stored d(pre_l) [h_used^2][n_pad][C_out]:
    -> [in_raster^2][n][c_in] (zero outside the consumed h_in x h_in window), sum |a||w|."""
    L = net.layers[l]
    hu, h_in, r = L["h_used"], L["h_in"], L["in_raster"]
    d = to_nhwc(dout_store, n, hu, L["c_out"])
    full = torch.zeros(n, 2 * h_in, 2 * h_in, L["c_out"], dtype=torch.float64, device=d.device)
    full[:, :hu, :hu] = d
    afull = full.abs()
    g = deconv_dinput(full, net.w[l])
    ag = deconv_dinput(afull, net.w[l].abs())
    out = torch.zeros(n, r, r, L["c_in"], dtype=torch.float64, device=d.device)
    aout = torch.zeros_like(out)
    out[:, :h_in, :h_in] = g
    aout[:, :h_in, :h_in] = ag
    return from_nhwc(out), from_nhwc(aout)


def linear_bwd_ref(net, dout_store, n, parts):
    """Linear backward from the stored d(pre_0) [16][n_pad][c4]: -> parts [parts][n][latent] (pixels 16/parts each)."""
    L = net.layers[0]
    c = L["c_out"]
    d = dout_store[:, :n, :c].double()                          # [16][n][c]
    W = net.w[0].reshape(L["c_in"], 16, c).permute(1, 2, 0)    # [16][c][latent]
    per = 16 // parts
    g = torch.stack([sum(d[q] @ W[q] for q in range(p * per, (p + 1) * per)) for p in range(parts)])
    ag = torch.stack([sum(d[q].abs() @ W[q].abs() for q in range(p * per, (p + 1) * per)) for p in range(parts)])
    return g, ag


def act_fwd(net, pre):
    if net.act == "sigmoid":
        y = torch.sigmoid(pre)
        return y, y * (1 - y)
    y = torch.tanh(pre)
    return y, 1 - y * y


def last_fwd_ref(net, x_store, n, bias=True):
    """The last layer's pre-activation [n][2fh][2fh][C] from its stored input [fh^2][n_pad][c1], and sum |a||w|."""
    x = to_nhwc(x_store, n, net.fh, net.layers[-1]["c_out"])
    f, b = net.w[-1], net.b[-1]
    return deconv(x, f, b if bias else None), deconv(x.abs(), f.abs(), b.abs() if bias else None)


def last_bwd_ref(net, dpre_nhwc):
    """d(act_{nl-1}) [fh^2][n][c1] from the last layer's d(pre) [n][2fh][2fh][C]."""
    return from_nhwc(deconv_dinput(dpre_nhwc, net.w[-1])), from_nhwc(deconv_dinput(dpre_nhwc.abs(), net.w[-1].abs()))


def bn_ref(net, l, pre, n):
    """act = relu(BN_batchstat(pre)) over the real rows [P][n][c] in fp64, and the size of the normalised terms."""
    off, sc = net.bn[l]
    c = net.layers[l]["c_out"]
    off, sc = off.reshape(-1, c) if l == 0 else off.reshape(1, c), sc.reshape(-1, c) if l == 0 else sc.reshape(1, c)
    off, sc = off.unsqueeze(1), sc.unsqueeze(1)                 # [P or 1][1][c]
    axes = (1,) if l == 0 else (0, 1)
    mean = pre.mean(dim=axes, keepdim=True)
    var = ((pre - mean) ** 2).mean(dim=axes, keepdim=True)
    inv = torch.rsqrt(var + 1e-5) * sc
    out = pre * inv + (off - mean * inv)
    size = (pre.abs() + mean.abs()) * inv.abs() + off.abs()
    return torch.relu(out), size




def bn_linear_ref(net, l, ws, raw, delta, n, tangent):
    """A BatchNorm layer's backward (tangent = False: d(act) -> d(pre), through the ReLU and the batch statistics) or
    tangent (True: t(pre) -> t(act)) on the exact GEMM output `raw` [P][n][c] that the kernel rounded by at most `delta`
    before the BatchNorm kernels read it in place.  Statistics over the real rows of the stored pre-activations; the mask
    is the stored activation > 0.  Returns the reference and its bound: delta carried through the (linear) map, plus the
    fp32 arithmetic of the BatchNorm kernels (partial sums of M / (8 * 16) terms each)."""
    tc = net.precision == "fp16"
    c = net.layers[l]["c_out"]
    pre = ws[("pre_h.%d" if tc else "pre.%d") % l][:, :n, :c].double()
    m = (ws[("act_h.%d" if tc else "act.%d") % l][:, :n, :c] > 0).double()
    sc = net.bn[l][1].reshape(-1, c) if l == 0 else net.bn[l][1].reshape(1, c)
    sc = sc.unsqueeze(1)
    axes = (1,) if l == 0 else (0, 1)
    M = n if l == 0 else n * pre.shape[0]
    mean = pre.mean(dim=axes, keepdim=True)
    inv = torch.rsqrt(((pre - mean) ** 2).mean(dim=axes, keepdim=True) + 1e-5)
    xh = (pre - mean) * inv
    k = (sc * inv).abs()
    dy, dl = (raw, delta) if tangent else (raw * m, delta * m)
    mu = lambda t: t.mean(dim=axes, keepdim=True)
    out = sc * inv * (dy - mu(dy) - xh * mu(dy * xh))
    bound = k * (dl + mu(dl) + xh.abs() * mu(dl * xh.abs()))
    bound = bound + k * (2.0 ** -20 * dy.abs() + (2.0 ** -18 + 2.0 ** -24 * (M / 128 + 64)) * (mu(dy.abs()) + xh.abs() * mu((dy * xh).abs())))
    if tangent:
        out, bound = out * m, bound * m
    return out, bound


def _into(net, ws, j, n, ref, ab, gamma, name, stats, tag, tangent=False):
    """Check the stored output of a GEMM into layer j's output (d(act_j), or the tangent of act_j): masked by layer j's
    stored ReLU mask, or through its BatchNorm, or neither (no activation)."""
    tc = net.precision == "fp16"
    out_t = "f16" if tc else "f32"
    L = net.layers[j]
    c = L["c_out"]
    got = ws[("dact_h.%d" if tc else "dact.%d") % j]
    if L["bn"]:
        delta = (half_ulp(ref, "f16") if tc else 0) + gamma * ab
        r, bound = bn_linear_ref(net, j, ws, ref, delta, n, tangent)
        check_close(tag + name + " + BN", got[:, :n, :c], r, torch.zeros_like(r), 0.0, out_t, stats, extra=bound)
        if bool((got[:, n:] != 0).any()):
            raise AssertionError(tag + name + " + BN: a tile-padding row is not 0")
    else:
        if L["relu"]:
            m = unpack_mask(ws["mask.%d" % j], L["c_out_p"])[:, :n] if tc else ws["act.%d" % j][:, :n] > 0
            ref, ab = ref * m[..., :c], ab * m[..., :c]
        check_close(tag + name, got[:, :n, :c], ref, ab, gamma, out_t, stats)
    check_zero_pad(tag + name, got, c)


def check_forward(net, ws, n, stats, tag, skip=()):
    """Every forward layer-direction of a call that ran the forward with masks (dgan_loss_grad, dgan_vjp, dgan_jvp):
    the GEMM layers (with BatchNorm: pre as a GEMM, act as the BatchNorm of the stored pre) and their masks."""
    tc = net.precision == "fp16"
    out_t = "f16" if tc else "f32"
    for l, L in enumerate(net.layers):
        name = "%s.fwd" % L["name"]
        if name in skip:
            continue
        x_store = ws["z_h" if tc else "z"] if l == 0 else ws[("act_h.%d" if tc else "act.%d") % (l - 1)]
        if l == 0:
            pre, ab = linear_fwd_ref(net, x_store.unsqueeze(0), n)
        else:
            pre, ab = deconv_fwd_ref(net, l, x_store, n)
        gamma = net.gamma(net.pairs(l, "fwd"), L["c_in_p"])
        c = L["c_out"]
        act_store = ws[("act_h.%d" if tc else "act.%d") % l]
        if L["bn"]:
            pre_store = ws[("pre_h.%d" if tc else "pre.%d") % l]
            check_close(tag + name + " (pre)", pre_store[:, :n, :c], pre, ab, gamma, "f32", stats)
            a_ref, size = bn_ref(net, l, pre_store[:, :n, :c].double(), n)
            check_close(tag + name + " (BN act)", act_store[:, :n, :c], a_ref, size, 2.0 ** -16, out_t, stats)
            check_zero_pad(tag + name + " pre", pre_store, c)
        else:
            ref = torch.relu(pre) if L["relu"] else pre
            check_close(tag + name, act_store[:, :n, :c], ref, ab, gamma, out_t, stats)
            if tc and L["relu"]:
                m = unpack_mask(ws["mask.%d" % l], L["c_out_p"])
                check_mask(tag + name, m[:, :n, :c], pre, gamma * ab)
                check_zero_pad(tag + name + " mask", m, c)
        check_zero_pad(tag + name + " act", act_store, c)


def check_last_y(net, ws, n, stats, tag):
    """The last layer's output y = act(pre) [n][2fh][2fh][C] from its stored input, to the activation's slope times the
    accumulation bound plus the activation's own error.  Returns the reference y, act'(y) and that bound."""
    tc = net.precision == "fp16"
    L = net.layers[-1]
    x_store = ws[("act_h.%d" if tc else "act.%d") % (net.nl - 1)]
    pre, ab = last_fwd_ref(net, x_store, n)
    gamma = net.gamma(net.pairs(net.nl, "fwd"), L["c_out_p"])
    y, dact = act_fwd(net, pre)
    dy = dact * gamma * ab + ACT_EPS[net.precision]            # |y - y_ref|
    w_out = 2 * net.fh
    C = net.c_img
    check_close(tag + "last.fwd (y)", ws["y"][:n].reshape(n, w_out, w_out, C), y, torch.zeros_like(y), 0.0, "f32", stats,
                extra=dy, where=["row", "i", "j", "c"])
    return y, dact, dy


def check_last_fwd(net, ws, n, x_img_rows, stats, tag):
    """The last layer's forward: y, the loss part of each 4x4 block (tensor cores) and the scaled d(pre) it stores
    (tensor cores: dblk = RN16(gscale * (y - x) * act'(y)); CUDA cores: dpre = (y - x) * act'(y))."""
    tc = net.precision == "fp16"
    y, dact, dy = check_last_y(net, ws, n, stats, tag)
    w_out = 2 * net.fh
    C = net.c_img
    x = x_img_rows.double().reshape(n, w_out, w_out, C)
    d = (y - x) * dact
    # d/dy of (y - x) act'(y) is at most 1.25 (sigmoid) or 5 (tanh) in magnitude
    dd = dy * (1.25 if net.act == "sigmoid" else 5.0)
    if tc:
        got = blocks_to_nhwc(ws["dblk"], n, w_out, C)
        check_close(tag + "last.fwd (dblk)", got, GRAD_SCALE * d, torch.zeros_like(d), 0.0, "f16", stats,
                    extra=GRAD_SCALE * dd, where=["row", "i", "j", "c"])
        # loss part of block (by, bx): sum over its 16 pixels of (y - x)^2
        e = (y - x) ** 2
        nb = w_out // 4
        lp = e.reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        tol = ((2 * (y - x).abs() + dy) * dy).reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        check_close(tag + "last.fwd (loss part)", ws["loss_part"][:, :n], lp, torch.zeros_like(lp), 0.0, "f32", stats,
                    extra=tol + 2.0 ** -20 * lp, where=["block", "row"])
    else:
        got = ws["dpre"][:n].reshape(n, w_out, w_out, C)
        check_close(tag + "last.fwd (dpre)", got, d, torch.zeros_like(d), 0.0, "f32", stats, extra=dd,
                    where=["row", "i", "j", "c"])


def stored_dpre(net, ws, n):
    """The last layer's d(pre) as its backward read it: [n][2fh][2fh][C] fp64."""
    w_out = 2 * net.fh
    if net.precision == "fp16":
        return blocks_to_nhwc(ws["dblk"], n, w_out, net.c_img)
    return ws["dpre"][:n].double().reshape(n, w_out, w_out, net.c_img)


def check_linear_bwd(net, ws, n, stats, tag):
    """The Linear's backward into z: its partial sums (tensor cores: 4 pixels each) from the stored d(pre_0)."""
    tc = net.precision == "fp16"
    g, ag = linear_bwd_ref(net, ws["dact_h.0" if tc else "dact.0"], n, LINEAR_SPLIT if tc else 1)
    lat = net.latent
    check_close(tag + "Linear.bwd", ws["g"][:, :n, :lat], g, ag, net.gamma(net.pairs(0, "bwd"), net.layers[0]["c_out_p"]),
                "f32", stats, where=["part", "row", "channel"])
    check_zero_pad(tag + "Linear.bwd", ws["g"], lat)


def check_backward(net, ws, n, stats, tag):
    """Every backward layer-direction: the last layer's and each GEMM layer's into its input (masked by the stored ReLU
    mask of that input, or through its BatchNorm backward, which overwrites the GEMM's output in place), the Linear's into
    z."""
    tc = net.precision == "fp16"
    nl = net.nl
    ref, ab = last_bwd_ref(net, stored_dpre(net, ws, n))
    K = 16 * net.c_img if tc else net.c_img
    _into(net, ws, nl - 1, n, ref, ab, net.gamma(net.pairs(nl, "bwd"), K), "last.bwd", stats, tag)
    for l in range(nl - 1, 0, -1):
        L = net.layers[l]
        ref, ab = deconv_bwd_ref(net, l, ws[("dact_h.%d" if tc else "dact.%d") % l], n)
        _into(net, ws, l - 1, n, ref, ab, net.gamma(net.pairs(l, "bwd"), L["c_out_p"]), "%s.bwd" % L["name"], stats, tag)
    check_linear_bwd(net, ws, n, stats, tag)


def check_inputs(net, ws, n, z):
    """z, v and z_h at the padded latent width: z = the caller's z, z_h = RN16(z), padded channels 0."""
    lat = net.latent
    assert torch.equal(ws["z"][:n, :lat], z), "z is not the caller's z"
    check_zero_pad("z", ws["z"], lat)
    check_zero_pad("v", ws["v"], lat)
    if net.precision == "fp16":
        assert torch.equal(ws["z_h"][:n, :lat], z.half()), "z_h is not RN16(z)"
        check_zero_pad("z_h", ws["z_h"], lat)


def check_row_scales(name, s, m, top, shared):
    """Power-of-two row scales (kernels_vjp.cuh pow2_scale): m * s in [2^(top-1), 2^top), one scale for all rows when
    shared (BatchNorm), 1 for a row whose m is 0.  m: the fp64 row maxima (the kernel's are fp32: ends get a 2^-20 slack)."""
    s, m = s.double(), m.double()
    if shared:
        m = m.max().expand_as(m)
    ok = (torch.frexp(s).mantissa == 0.5) & torch.where(
        m > 0, (m * s >= 2.0 ** (top - 1) * (1 - 2.0 ** -20)) & (m * s < 2.0 ** top * (1 + 2.0 ** -20)), s == 1)
    if not bool(ok.all()):
        r = int(torch.nonzero(~ok)[0])
        raise AssertionError("%s: row %d has scale %r for a row maximum %r" % (name, r, float(s[r]), float(m[r])))


def check_pad_rows_zero(name, buf, n, row_axis=0):
    """Every tile-padding row (index >= n along row_axis) of buf is exactly 0; the failure names the first such row."""
    tail = buf.narrow(row_axis, n, buf.shape[row_axis] - n)
    if tail.numel() and bool((tail != 0).any()):
        idx = [int(i) for i in torch.nonzero(tail != 0)[0]]
        raise AssertionError("%s: tile-padding row %d is not 0 (%r)" % (name, n + idx[row_axis], float(tail[tuple(idx)])))


def check_cotangent(net, ws, n, dy, stats, tag, scale="loss"):
    """dgan_vjp's entry: d(pre) = dy * act'(y) from the stored y; tensor cores: scaled by the power-of-two row scales it
    keeps in the workspace buffer `scale` (`loss` for dgan_vjp, `mscale` for the measured entries, whose `loss` holds the
    loss) with max |d(pre)| * s in [8, 16), into the block tensor, the tile-padding rows 0; CUDA cores: unscaled in dpre,
    the tile-padding rows 0."""
    w_out = 2 * net.fh
    C = net.c_img
    y = ws["y"][:n].double()
    d = dy.reshape(n, -1).double() * (y * (1 - y) if net.act == "sigmoid" else 1 - y * y)
    if net.precision == "fp16":
        s = ws[scale][:n]
        check_row_scales(tag + "cotangent (row scales)", s, d.abs().amax(dim=1), 4, net.use_bn)
        ref = (d * s.double().unsqueeze(1)).reshape(n, w_out, w_out, C)
        got = blocks_to_nhwc(ws["dblk"], n, w_out, C)
        check_close(tag + "cotangent (dblk)", got, ref, torch.zeros_like(ref), 0.0, "f16", stats,
                    extra=2.0 ** -21 * ref.abs(), where=["row", "i", "j", "c"])
        check_pad_rows_zero(tag + "cotangent (dblk)", ws["dblk"], n, row_axis=1)
    else:
        ref = d.reshape(n, w_out, w_out, C)
        got = ws["dpre"][:n].reshape(n, w_out, w_out, C)
        check_close(tag + "cotangent (dpre)", got, ref, torch.zeros_like(ref), 0.0, "f32", stats,
                    extra=2.0 ** -21 * ref.abs(), where=["row", "i", "j", "c"])
        check_pad_rows_zero(tag + "cotangent (dpre)", ws["dpre"], n)


def check_measured_loss(ws, n, m, stats, tag):
    """The measured loss of each real row from the stored residuals r [n_pad][m_ld]: loss = (1/m) sum_j r_j^2 (the
    kernels' fp32 squares, one partial per 64-column tile, the tiles summed in a fixed order, times fl(1/m)), within
    (m + 3) u of the fp64 value: any order of m non-negative terms, the squares' roundings and the two of the multiply."""
    r = ws["r"][:n].double()
    ref = (r * r).sum(dim=1) / m
    check_close(tag + "measured loss", ws["loss"][:n], ref, torch.zeros_like(ref), 0.0, "f32", stats,
                extra=(m + 3) * 2.0 ** -24 * ref, where=["row"])


def check_tangent(net, ws, n, t, ty, stats, tag):
    """dgan_jvp's tangent pass, after a forward that kept its masks: the tangent of z enters (tensor cores: z_h =
    RN16(t * s_n) with power-of-two row scales in `loss`, max |t| * s in [0.25, 0.5); CUDA cores: v = t); each layer's
    tangent direction (forward weights, no bias) on its stored input, masked by the primal forward's masks or through the
    BatchNorm tangent; the last layer's fp32 tangent of pre (tensor cores: the block tensor in dpre); and
    ty = t(pre) * act'(y) / s_n from the stored t(pre) and y."""
    tc = net.precision == "fp16"
    lat = net.latent
    if tc:
        s = ws["loss"][:n]
        check_row_scales(tag + "tangent (row scales)", s, t.abs().amax(dim=1), -1, net.use_bn)
        assert torch.equal(ws["z_h"][:n, :lat], (t * s.unsqueeze(1)).half()), "z_h is not RN16(t * s)"
        assert not bool((ws["z_h"][n:] != 0).any()), "a tile-padding row of z_h is not 0"
        check_zero_pad("z_h", ws["z_h"], lat)
    else:
        s = torch.ones(n, dtype=torch.float32, device=t.device)
        assert torch.equal(ws["v"][:n, :lat], t), "v is not the tangent"
        assert not bool((ws["v"][n:] != 0).any()), "a tile-padding row of v is not 0"
        check_zero_pad("v", ws["v"], lat)
    for l, L in enumerate(net.layers):
        x_store = ws["z_h" if tc else "v"] if l == 0 else ws[("dact_h.%d" if tc else "dact.%d") % (l - 1)]
        if l == 0:
            ref, ab = linear_fwd_ref(net, x_store.unsqueeze(0), n, bias=False)
        else:
            ref, ab = deconv_fwd_ref(net, l, x_store, n, bias=False)
        _into(net, ws, l, n, ref, ab, net.gamma(net.pairs(l, "fwd"), L["c_in_p"]), "%s.jvp" % L["name"], stats, tag,
              tangent=True)
    w_out = 2 * net.fh
    C = net.c_img
    ref, ab = last_fwd_ref(net, ws[("dact_h.%d" if tc else "dact.%d") % (net.nl - 1)], n, bias=False)
    if tc:
        # dpre holds the fp32 block tensor [n_blocks][n_pad][16 C] (as many elements as [n_pad][H W C])
        got = blocks_to_nhwc(ws["dpre"].reshape((w_out // 4) ** 2, -1, 16 * C), n, w_out, C)
    else:
        got = ws["dpre"][:n].reshape(n, w_out, w_out, C)
    check_close(tag + "last.jvp", got, ref, ab, net.gamma(net.pairs(net.nl, "fwd"), net.layers[-1]["c_out_p"]), "f32", stats,
                where=["row", "i", "j", "c"])
    y = ws["y"][:n].double().reshape(n, w_out, w_out, C)
    want = got.double() * (y * (1 - y) if net.act == "sigmoid" else 1 - y * y) / s.double().reshape(n, 1, 1, 1)
    check_close(tag + "ty", ty.reshape(n, w_out, w_out, C), want, torch.zeros_like(want), 0.0, "f32", stats,
                extra=2.0 ** -21 * want.abs() + 2.0 ** -140, where=["row", "i", "j", "c"])


def check_momentum(net, ws, z0, lr, mu, hwc, stats, tag):
    """The momentum update after one step from v = 0 (dgan_reconstruct with L = 2 leaves the first step's partial sums in
    g and the updated z, v, z_h): v = fl(gmul * sum of the parts in order), z = z0 - lr * v, to 2 fp32 ulps; z_h = RN16(z)
    exactly; the tail's tile counters are back at 0.  gmul = 2 / HWC (tensor cores: / grad_scale)."""
    tc = net.precision == "fp16"
    g = ws["g"]
    gs = g[0].clone()
    for p in range(1, g.shape[0]):
        gs = gs + g[p]
    gmul = torch.tensor(2.0, dtype=torch.float32) / torch.tensor(float(hwc), dtype=torch.float32)
    if tc:
        gmul = gmul / torch.tensor(GRAD_SCALE, dtype=torch.float32)
    v_ref = (gmul.to(gs.device) * gs).double()
    v = ws["v"].double()
    check_close(tag + "momentum (v)", v, v_ref, torch.zeros_like(v), 0.0, "f32", stats,
                extra=4 * half_ulp(v_ref, "f32") + 2.0 ** -149, where=["row", "channel"])
    zp = torch.zeros_like(ws["z"])
    zp[:z0.shape[0], :z0.shape[1]] = z0
    z_ref = zp.double() - lr * v
    check_close(tag + "momentum (z)", ws["z"], z_ref, torch.zeros_like(z_ref), 0.0, "f32", stats,
                extra=4 * (half_ulp(z_ref, "f32") + half_ulp(lr * v, "f32")), where=["row", "channel"])
    check_zero_pad(tag + "momentum (z)", ws["z"], net.latent)
    check_zero_pad(tag + "momentum (v)", ws["v"], net.latent)
    if tc:
        assert torch.equal(ws["z_h"], ws["z"].half()), "z_h is not RN16(z) after the update"
        assert not bool((ws["mom_counter"] != 0).any()), "the momentum tail's tile counters are not back at 0"


def check_momentum_rows(net, ws, z0, lr, mu, n, stats, tag):
    """momentum_rows_kernel (the measured loop's update) after one step from v = 0 (dgan_reconstruct_measured with L = 2
    leaves the first step's partial sums in g, its row scales in mscale and the updated z, v, z_h): on the real rows
    v = fl(sum of the parts in order) / mscale[row] (tensor cores: power-of-two scales, so the division is exact) or
    unscaled (CUDA cores), z = z0 - lr * v, both to check_momentum's bound; the tile-padding rows and padded latent
    channels of v and z exactly 0; z_h = RN16(z) exactly; the split-K tail's counters untouched (0: the measured loop
    does not run the tail).  mu, the call's momentum, does not enter a step from v = 0."""
    tc = net.precision == "fp16"
    lat = net.latent
    g = ws["g"]
    gs = g[0].clone()
    for p in range(1, g.shape[0]):
        gs = gs + g[p]
    v_ref = gs[:n, :lat].double()
    if tc:
        v_ref = v_ref / ws["mscale"][:n].double().unsqueeze(1)
    v = ws["v"]
    check_close(tag + "momentum rows (v)", v[:n, :lat], v_ref, torch.zeros_like(v_ref), 0.0, "f32", stats,
                extra=4 * half_ulp(v_ref, "f32") + 2.0 ** -149, where=["row", "channel"])
    z_ref = z0[:n, :lat].double() - lr * v[:n, :lat].double()
    check_close(tag + "momentum rows (z)", ws["z"][:n, :lat], z_ref, torch.zeros_like(z_ref), 0.0, "f32", stats,
                extra=4 * (half_ulp(z_ref, "f32") + half_ulp(lr * v[:n, :lat].double(), "f32")), where=["row", "channel"])
    for nm in ("v", "z"):
        check_pad_rows_zero(tag + "momentum rows (%s)" % nm, ws[nm], n)
        check_zero_pad(tag + "momentum rows (%s)" % nm, ws[nm], lat)
    if tc:
        if not torch.equal(ws["z_h"], ws["z"].half()):
            r = int(torch.nonzero(ws["z_h"] != ws["z"].half())[0][0])
            raise AssertionError(tag + "momentum rows (z_h): row %d is not RN16(z)" % r)
        assert not bool((ws["mom_counter"] != 0).any()), tag + "momentum rows: the split-K tail's counters are not 0"
