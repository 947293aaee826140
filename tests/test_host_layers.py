"""CPU tests (no GPU) of the per-layer checker of test_gpu_layers.py (tests/layer_ref.py): it accepts an emulation of
the tensor-core path's loss gradient, vjp, jvp and momentum update (MNIST, latent 64 / net_dim 32, 300 rows in two 256-row
tile pairs) that accumulates in fp32 in another order with the kernels' rounding points, and it rejects that emulation
with one defect seeded into one layer-direction - one (input pixel, tap) product dropped, one 64-channel k-chunk dropped
(where K has more than one), a column block shifted by 64 channels, one ReLU mask bit flipped where |pre| is not tiny,
the bias omitted, two 128-row tiles swapped, the gradient or cotangent row scale off by 2, the momentum multiplier off by
2 or a partial sum missing - in every layer-direction kind the defect applies to.  That is what shows the bound is tight
enough to matter.  The BatchNorm, CelebA, column-block and fp32 variants of the same checks run on the GPU only."""
import pytest
import torch

import layer_ref as R
from oracle import defensegan_oracle as O

ARCH, LATENT, NET_DIM, N_ROWS, N_PAD = "mnist", 64, 32, 300, 512
PADDED = [64, 256, 64, 64]           # the fp16 width rule at latent 64, net_dim 32


def _deconv_fwd_pairs(h_in, h_used, raster):
    """[(input pixel, ka, kb)] per output pixel of a 5x5 / stride-2 transposed conv (pixel-graph order)."""
    out = []
    for i in range(h_used):
        for j in range(h_used):
            lst = []
            for ka in range(5):
                oo = i + 1 - ka
                if oo < 0 or oo % 2 or oo // 2 >= h_in:
                    continue
                for kb in range(5):
                    pp = j + 1 - kb
                    if pp < 0 or pp % 2 or pp // 2 >= h_in:
                        continue
                    lst.append(((oo // 2) * raster + pp // 2, ka, kb))
            out.append(lst)
    return out


def _deconv_bwd_pairs(h_in, h_used, raster):
    """[(output pixel, ka, kb)] per input raster pixel."""
    out = []
    for o in range(raster):
        for p in range(raster):
            lst = []
            for ka in range(5):
                i = 2 * o + ka - 1
                if o >= h_in or p >= h_in or i < 0 or i >= h_used:
                    continue
                for kb in range(5):
                    j = 2 * p + kb - 1
                    if 0 <= j < h_used:
                        lst.append((i * h_used + j, ka, kb))
            out.append(lst)
    return out


def _pack(bits):
    sh = torch.arange(64, dtype=torch.int64)
    P, n, c = bits.shape
    return (bits.reshape(P, n, c // 64, 64).long() << sh).sum(-1)


class Emu:
    """An fp32-accumulating CPU emulation of dgan_loss_grad on the tensor-core path, writing the buffers the kernels
    write.  defect = (layer-direction, kind) seeds one defect into one layer-direction."""

    def __init__(self, defect=None):
        self.defect = defect
        self.w = O.init_generator_weights(ARCH, latent_dim=LATENT, net_dim=NET_DIM, random_bias=True)
        self.net = R.Net(ARCH, LATENT, NET_DIM, False, "fp16", PADDED, self.w, torch.device("cpu"))
        g = torch.Generator().manual_seed(1)
        self.z = torch.randn(N_ROWS, LATENT, generator=g) * LATENT ** -0.5
        self.x = torch.rand(N_ROWS, 28 * 28, generator=g)

    def _d(self, name, kind):
        return self.defect is not None and self.defect == (name, kind)

    def gemm(self, name, inp, pairs, weight, n_out):
        """acc[q] = sum over the pairs of q of inp[p] @ weight(pair), fp32, with the pair / k-chunk defects."""
        P_in, n, K = inp.shape
        acc = torch.zeros(len(pairs), n, n_out)
        a = inp.float()
        for q, lst in enumerate(pairs):
            for i, pr in enumerate(lst):
                wm = weight(pr).float()                          # [K][n_out]
                contrib = a[pr[0]] @ wm
                if q == len(pairs) // 2 and i == 0:
                    if self._d(name, "drop_pair"):
                        contrib[:128] = 0
                    elif self._d(name, "drop_kchunk"):
                        contrib[:128] = a[pr[0], :128, 64:] @ wm[64:]
                acc[q] += contrib
        if self._d(name, "shift64"):
            acc[..., 64:] = acc[..., :-64].clone()
            acc[..., :64] = 0
        if self._d(name, "swap_tiles"):
            acc[:, :256] = torch.cat([acc[:, 128:256], acc[:, :128]], dim=1)
        return acc

    def flip(self, name, m, val):
        """Flip the mask bit of the largest |val| of row 5 (a mask defect)."""
        if self._d(name, "mask"):
            q, c = divmod(int(val[:, 5].abs().argmax()), val.shape[2])
            m[q, 5, c] = ~m[q, 5, c]
        return m

    def run(self):
        net, ws = self.net, {}
        lat_p, c4p, c2p, c1p = PADDED
        z = torch.zeros(N_PAD, lat_p)
        z[:N_ROWS, :LATENT] = self.z
        ws["z"], ws["v"], ws["z_h"] = z, torch.zeros_like(z), z.half()
        pad = lambda t, r, c: torch.nn.functional.pad(t, (0, c - t.shape[-1], 0, r - t.shape[-2]))
        W0 = pad(torch.as_tensor(self.w["Generator.Input/Generator.Input.W"]).half(), lat_p, 16 * 4 * NET_DIM)
        W0 = W0.reshape(lat_p, 16, 4 * NET_DIM)
        W0 = torch.nn.functional.pad(W0, (0, c4p - 4 * NET_DIM))          # [lat_p][16][c4p]
        b0 = torch.nn.functional.pad(torch.as_tensor(self.w["Generator.Input/Generator.Input.b"]).reshape(16, -1),
                                     (0, c4p - 4 * NET_DIM))
        masks = []
        self.W0, self.masks = W0, masks
        # ---- forward
        acc = self.gemm("Linear.fwd", ws["z_h"].unsqueeze(0), [[(0, q)] for q in range(16)], lambda pr: W0[:, pr[1]], c4p)
        pre = acc + (0 if self._d("Linear.fwd", "bias") else b0.unsqueeze(1))
        m = self.flip("Linear.fwd", pre > 0, pre)
        masks.append(m)
        ws["act_h.0"], ws["mask.0"] = torch.relu(pre).half(), _pack(m)
        specs = [("Generator.2", 4, 7, 4, c4p, c2p), ("Generator.3", 7, 14, 7, c2p, c1p)]
        filt = {}
        for l, (nm, h_in, hu, r, cin, cout) in enumerate(specs, start=1):
            F = torch.as_tensor(self.w["%s/%s.Filters" % (nm, nm)]).half()       # (5, 5, C_out, C_in)
            b = torch.as_tensor(self.w["%s/%s.Biases" % (nm, nm)])
            b = torch.nn.functional.pad(b, (0, cout - b.shape[0]))
            F = torch.nn.functional.pad(F, (0, cin - F.shape[3], 0, cout - F.shape[2]))
            filt[nm] = F
            acc = self.gemm(nm + ".fwd", ws["act_h.%d" % (l - 1)], _deconv_fwd_pairs(h_in, hu, r),
                            lambda pr, F=F: F[pr[1], pr[2]].t(), cout)
            pre = acc + (0 if self._d(nm + ".fwd", "bias") else b)
            m = self.flip(nm + ".fwd", pre > 0, pre)
            masks.append(m)
            ws["act_h.%d" % l], ws["mask.%d" % l] = torch.relu(pre).half(), _pack(m)
        self.filt, self.specs = filt, specs
        # the last layer in image space (the kernel works on 4x4 blocks of it: the same products)
        F5 = torch.nn.functional.pad(torch.as_tensor(self.w["Generator.5/Generator.5.Filters"]).half(), (0, c1p - NET_DIM))
        self.F5 = F5
        b5 = torch.as_tensor(self.w["Generator.5/Generator.5.Biases"])
        acc = self.gemm("last.fwd", ws["act_h.2"], _deconv_fwd_pairs(14, 28, 14), lambda pr: F5[pr[1], pr[2]].t(), 1)
        pre = acc + (0 if self._d("last.fwd", "bias") else b5)                        # [784][n_pad][1]
        y = torch.sigmoid(pre)
        xr = torch.zeros(N_PAD, 784)
        xr[:N_ROWS] = self.x
        xr[N_ROWS:] = self.x[-1]
        d = y - xr.t().unsqueeze(-1)
        gs = R.GRAD_SCALE * (2 if self._d("last.fwd", "gscale") else 1)
        dpre = (d * y * (1 - y) * gs).half()                                             # [784][n_pad][1]
        ws["y"] = y[:, :, 0].t().contiguous()
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dblk = torch.zeros(49, N_PAD, 16, dtype=torch.float16)
        dblk[blk, :, k] = dpre[:, :, 0]
        ws["dblk"] = dblk
        lp = torch.zeros(49, N_PAD)
        lp.index_add_(0, blk, (d[:, :, 0] ** 2))
        ws["loss_part"] = lp
        self.backward(ws)
        return ws

    def backward(self, ws):
        """The backward layer-directions from the stored dblk."""
        lat_p, c4p, c2p, c1p = PADDED
        F5, W0, masks, specs, filt = self.F5, self.W0, self.masks, self.specs, self.filt
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dimg = ws["dblk"][blk, :, k].unsqueeze(-1)                                             # [784][n_pad][1] as read
        acc = self.gemm("last.bwd", dimg, _deconv_bwd_pairs(14, 28, 14), lambda pr: F5[pr[1], pr[2]], c1p)
        m = self.flip("last.bwd", masks[2].clone(), acc)
        ws["dact_h.2"] = (acc * m).half()
        for l, (nm, h_in, hu, r, cin, cout) in reversed(list(enumerate(specs, start=1))):
            F = filt[nm]
            acc = self.gemm(nm + ".bwd", ws["dact_h.%d" % l], _deconv_bwd_pairs(h_in, hu, r), lambda pr, F=F: F[pr[1], pr[2]],
                            cin)
            m = self.flip(nm + ".bwd", masks[l - 1].clone(), acc)
            ws["dact_h.%d" % (l - 1)] = (acc * m).half()
        parts = []
        for p in range(R.LINEAR_SPLIT):
            parts.append(self.gemm("Linear.bwd", ws["dact_h.0"][4 * p:4 * p + 4], [[(q, q) for q in range(4)]],
                                   lambda pr, p=p: W0[:, 4 * p + pr[1]].t(), lat_p)[0])
        ws["g"] = torch.stack(parts)

    def run_vjp(self, dy):
        """dgan_vjp after the forward of run(): the cotangent entry, then the backward."""
        ws = self.run()
        y = ws["y"][:N_ROWS]
        d = dy * (y * (1 - y))
        m = d.abs().amax(dim=1).double()
        s = torch.exp2(4 - torch.floor(torch.log2(m)) - 1).float()          # max |d| * s in [8, 16)
        ws["loss"] = torch.ones(N_PAD)
        ws["loss"][:N_ROWS] = s
        sd = d * s.unsqueeze(1) * (2 if self._d("cotangent", "gscale") else 1)
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dblk = torch.zeros(49, N_PAD, 16, dtype=torch.float16)
        dblk[blk, :N_ROWS, k] = sd.t().half()
        if self._d("cotangent", "swap_tiles"):
            dblk[:, :256] = torch.cat([dblk[:, 128:256], dblk[:, :128]], dim=1)
        ws["dblk"] = dblk
        self.backward(ws)
        return ws

    def run_jvp(self, t):
        """dgan_jvp after the forward of run(): the tangent entry, the tangent directions (masked by the primal masks), the
        last layer's fp32 tangent of pre as the block tensor in dpre, and ty."""
        ws = self.run()
        lat_p, c4p, c2p, c1p = PADDED
        s = torch.exp2(-1 - torch.floor(torch.log2(t.abs().amax(dim=1).double())) - 1).float()   # max |t| s in [0.25, 0.5)
        ws["loss"] = torch.ones(N_PAD)
        ws["loss"][:N_ROWS] = s
        zh = torch.zeros(N_PAD, lat_p, dtype=torch.float16)
        zh[:N_ROWS, :LATENT] = (t * s.unsqueeze(1)).half()
        ws["z_h"] = zh
        acc = self.gemm("Linear.jvp", zh.unsqueeze(0), [[(0, q)] for q in range(16)], lambda pr: self.W0[:, pr[1]], c4p)
        ws["dact_h.0"] = (acc * self.flip("Linear.jvp", self.masks[0].clone(), acc)).half()
        for l, (nm, h_in, hu, r, cin, cout) in enumerate(self.specs, start=1):
            F = self.filt[nm]
            acc = self.gemm(nm + ".jvp", ws["dact_h.%d" % (l - 1)], _deconv_fwd_pairs(h_in, hu, r),
                            lambda pr, F=F: F[pr[1], pr[2]].t(), cout)
            ws["dact_h.%d" % l] = (acc * self.flip(nm + ".jvp", self.masks[l].clone(), acc)).half()
        tp = self.gemm("last.jvp", ws["dact_h.2"], _deconv_fwd_pairs(14, 28, 14), lambda pr: self.F5[pr[1], pr[2]].t(), 1)
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dpre = torch.zeros(49, N_PAD, 16)
        dpre[blk, :, k] = tp[:, :, 0]
        ws["dpre"] = dpre.reshape(N_PAD, 784)
        y = ws["y"][:N_ROWS]
        ty = tp[:, :N_ROWS, 0].t() * (y * (1 - y)) / s.unsqueeze(1)
        return ws, ty

    def run_momentum(self, lr):
        """The momentum update from v = 0 on the partial sums of run()'s Linear backward."""
        ws = self.run()
        g = ws["g"]
        gs = g[0].clone()
        for p in range(1, g.shape[0] - (1 if self._d("momentum", "drop_part") else 0)):
            gs = gs + g[p]
        gmul = torch.tensor(2.0) / torch.tensor(784.0) / torch.tensor(R.GRAD_SCALE)
        v = gmul * gs * (2 if self._d("momentum", "gmul") else 1)
        z0 = ws["z"].clone()
        ws["v"], ws["z"] = v, z0 - lr * v
        ws["z_h"], ws["mom_counter"] = ws["z"].half(), torch.zeros(N_PAD // 128, dtype=torch.int32)
        return ws, z0[:N_ROWS, :LATENT]

    def check(self, ws):
        stats = R.Stats()
        R.check_inputs(self.net, ws, N_ROWS, self.z)
        R.check_forward(self.net, ws, N_ROWS, stats, "")
        R.check_last_fwd(self.net, ws, N_ROWS, self.x, stats, "")
        R.check_backward(self.net, ws, N_ROWS, stats, "")
        return stats


    def check_vjp(self, ws, dy):
        stats = R.Stats()
        R.check_forward(self.net, ws, N_ROWS, stats, "")
        R.check_cotangent(self.net, ws, N_ROWS, dy, stats, "")
        R.check_backward(self.net, ws, N_ROWS, stats, "")
        return stats

    def check_jvp(self, ws, t, ty):
        stats = R.Stats()
        R.check_forward(self.net, ws, N_ROWS, stats, "", skip=("Linear.fwd",))
        R.check_tangent(self.net, ws, N_ROWS, t, ty, stats, "")
        return stats

    def check_momentum(self, ws, z0, lr):
        stats = R.Stats()
        R.check_linear_bwd(self.net, ws, N_ROWS, stats, "")
        R.check_momentum(self.net, ws, z0, lr, 0.7, 784, stats, "")
        return stats


def _dy():
    return torch.randn(N_ROWS, 784, generator=torch.Generator().manual_seed(5)) * 0.3


def _t():
    return torch.randn(N_ROWS, LATENT, generator=torch.Generator().manual_seed(6)) * 3.0


def _run(emu, what):
    """Emulate call `what` and check it with the checker of that call."""
    if what == "loss_grad":
        return emu.check(emu.run())
    if what == "vjp":
        return emu.check_vjp(emu.run_vjp(_dy()), _dy())
    if what == "jvp":
        ws, ty = emu.run_jvp(_t())
        return emu.check_jvp(ws, _t(), ty)
    ws, z0 = emu.run_momentum(10.0)
    return emu.check_momentum(ws, z0, 10.0)


@pytest.mark.parametrize("what", ["loss_grad", "vjp", "jvp", "momentum"])
def test_checker_accepts_an_fp32_emulation(what):
    stats = _run(Emu(), what)
    print("\n" + "\n".join(stats.lines()))
    assert len(stats.rows) >= 2


# (call, layer-direction, defect)
DEFECTS = []
for _name in ["Linear.fwd", "Generator.2.fwd", "Generator.3.fwd", "last.fwd", "last.bwd", "Generator.3.bwd",
              "Generator.2.bwd", "Linear.bwd", "Linear.jvp", "Generator.2.jvp", "Generator.3.jvp", "last.jvp"]:
    for _kind in ["drop_pair", "drop_kchunk", "shift64", "mask", "bias", "swap_tiles", "gscale"]:
        if _kind == "bias" and not _name.endswith(".fwd") or _kind == "gscale" and _name != "last.fwd":
            continue
        if _kind == "mask" and _name in ("last.fwd", "Linear.bwd", "last.jvp"):     # no ReLU mask there
            continue
        if _kind == "shift64" and _name in ("last.fwd", "last.jvp"):                  # 16 output columns
            continue
        # K = 64 (one k-chunk: dropping it is dropping the pair) or K = 16 (the last layer's backward)
        if _kind == "drop_kchunk" and _name in ("Linear.fwd", "Generator.3.fwd", "last.fwd", "last.bwd", "Generator.3.bwd",
                                                 "Generator.2.bwd", "Linear.jvp", "Generator.3.jvp", "last.jvp"):
            continue
        DEFECTS.append(("jvp" if _name.endswith(".jvp") else "loss_grad", _name, _kind))
DEFECTS += [("vjp", "cotangent", "gscale"), ("vjp", "cotangent", "swap_tiles"), ("momentum", "momentum", "gmul"),
            ("momentum", "momentum", "drop_part")]


@pytest.mark.parametrize("what,name,kind", DEFECTS)
def test_checker_rejects_a_seeded_defect(what, name, kind):
    emu = Emu(defect=(name, kind))
    with pytest.raises(AssertionError, match=name.replace(".", r"\.")):
        _run(emu, what)
