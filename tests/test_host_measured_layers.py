"""CPU tests (no GPU) of the per-layer checks of the measured projection (tests/layer_ref.py check_last_y,
check_measured_loss, check_cotangent with the row scales in `mscale`, check_momentum_rows), run by
test_gpu_measured_layers.py on the workspace of dgan_loss_grad_measured and dgan_reconstruct_measured.  The input is
test_host_layers.py's fp32 emulation of the tensor-core path made measured: after its forward, the residuals
r = A G - y of a Gaussian sketch (m = 200, no multiple of the 64-column tile), the measured loss from one fp32 partial
per 64-column tile, the cotangent dy = (2/m) A^T r, the cotangent entry at the kernels' rounding points
(d(pre) = dy * act'(y) in fp32, times the power-of-two row scale, rounded to fp16; the scales in `mscale`, the measured
loss in `loss`), the backward, and momentum_rows_kernel's update (v = sum of the split-K parts / mscale[row] on the real
rows, z = z0 - lr v, z_h = RN16(z)).  The checks accept it and reject it with one defect seeded - one row's scale off by
2, each row divided by its neighbour's scale, a tile-padding row of dblk not 0, the update not dividing out one row's
scale, a split-K partial missing, a 64-column tile missing from the loss - each in a failure that names the
layer-direction and the row.  A scale applied to the tile-padding rows is harmful only where the never-written scale
there is 0 or NaN; the checks see it then, and it changes no bit otherwise."""
import re

import pytest
import torch

import layer_ref as R
from test_host_layers import Emu, N_PAD, N_ROWS

M = 200
M_LD = 256                           # m rounded up to the 64-column tile
LR = 10.0 * M / 784


class MeasuredEmu(Emu):
    """Emu with the measured loss: defect = (layer-direction, kind, row); pad_scale: what the never-written tile-padding
    rows of mscale hold."""

    def __init__(self, defect=None, pad_scale=0.0):
        super().__init__(defect[:2] if defect else None)
        g = torch.Generator().manual_seed(11)
        self.a = torch.randn(M, 784, generator=g) / 28.0
        self.ym = self.x @ self.a.t() + 0.01 * torch.randn(N_ROWS, M, generator=g)
        self.ym *= torch.exp2(torch.arange(N_ROWS) % 5.0).unsqueeze(1)     # residuals, so row scales, 2^0 .. 2^4 apart
        self.row = defect[2] if defect else None
        self.pad_scale = pad_scale

    def run_measured(self):
        """dgan_loss_grad_measured after the forward of run(): the two products and the measured loss, the cotangent
        entry with its row scales in mscale, the backward."""
        ws = self.run()
        y = ws["y"][:N_ROWS]
        r = y @ self.a.t() - self.ym
        ws["r"] = torch.zeros(N_PAD, M_LD)
        ws["r"][:N_ROWS, :M] = r
        parts = (ws["r"][:N_ROWS] ** 2).reshape(N_ROWS, M_LD // 64, 64).sum(dim=2)   # one partial per column tile
        if self._d("measured loss", "drop_tile"):
            parts[:, -1] = 0
        loss = parts[:, 0].clone()
        for t in range(1, M_LD // 64):
            loss = loss + parts[:, t]
        ws["loss"] = torch.zeros(N_PAD)
        ws["loss"][:N_ROWS] = loss * torch.tensor(1.0 / M)
        dy = torch.tensor(2.0 / M) * (r @ self.a)
        ws["dym"] = dy
        d = dy * (y * (1 - y))
        s = torch.exp2(4 - torch.floor(torch.log2(d.abs().amax(dim=1).double())) - 1).float()   # max |d| s in [8, 16)
        ws["mscale"] = torch.full((N_PAD,), self.pad_scale)          # the tile-padding rows are never written
        ws["mscale"][:N_ROWS] = s
        sd = d * s.unsqueeze(1)
        if self._d("cotangent", "row_scale"):
            sd[self.row] *= 2
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dblk = torch.zeros(49, N_PAD, 16, dtype=torch.float16)
        dblk[blk, :N_ROWS, k] = sd.t().half()
        if self._d("cotangent", "pad_row"):
            dblk[:, self.row] = dblk[:, 0]
        ws["dblk"] = dblk
        self.backward(ws)
        return ws

    def run_momentum_rows(self, lr):
        """momentum_rows_kernel from v = 0 after run_measured()."""
        ws = self.run_measured()
        g = ws["g"]
        gs = g[0].clone()
        for p in range(1, g.shape[0] - (1 if self._d("momentum rows", "drop_part") else 0)):
            gs = gs + g[p]
        gmul = torch.ones(N_PAD)
        gmul[:N_ROWS] = 1.0 / ws["mscale"][:N_ROWS]
        if self._d("momentum rows", "pad_scale"):
            gmul = 1.0 / ws["mscale"]
        if self._d("momentum rows", "wrong_row"):
            gmul[:N_ROWS - 1] = 1.0 / ws["mscale"][1:N_ROWS]
        if self._d("momentum rows", "unscaled_row"):
            gmul[self.row] = 1.0
        v = gmul.unsqueeze(1) * gs
        z0 = ws["z"].clone()
        ws["v"], ws["z"] = v, z0 - lr * v
        ws["z_h"], ws["mom_counter"] = ws["z"].half(), torch.zeros(N_PAD // 128, dtype=torch.int32)
        return ws, z0[:N_ROWS, :self.net.latent]

    def check_measured(self, ws, scale="mscale"):
        stats = R.Stats()
        R.check_inputs(self.net, ws, N_ROWS, self.z)
        R.check_forward(self.net, ws, N_ROWS, stats, "")
        R.check_last_y(self.net, ws, N_ROWS, stats, "")
        R.check_measured_loss(ws, N_ROWS, M, stats, "")
        R.check_cotangent(self.net, ws, N_ROWS, ws["dym"], stats, "", scale=scale)
        R.check_backward(self.net, ws, N_ROWS, stats, "")
        return stats

    def check_momentum_rows(self, ws, z0, lr):
        stats = R.Stats()
        R.check_linear_bwd(self.net, ws, N_ROWS, stats, "")
        R.check_momentum_rows(self.net, ws, z0, lr, 0.7, N_ROWS, stats, "")
        return stats


def _run(emu, what):
    if what == "loss_grad":
        return emu.check_measured(emu.run_measured())
    ws, z0 = emu.run_momentum_rows(LR)
    return emu.check_momentum_rows(ws, z0, LR)


@pytest.mark.parametrize("what", ["loss_grad", "momentum"])
def test_checker_accepts_a_measured_fp32_emulation(what):
    stats = _run(MeasuredEmu(), what)
    print("\n" + "\n".join(stats.lines()))
    want = ("cotangent (dblk)", "measured loss", "last.fwd (y)") if what == "loss_grad" else ("momentum rows (v)",)
    assert all(k in stats.rows for k in want)


def test_cotangent_check_reads_the_row_scales_where_it_is_told():
    """The measured entries keep the loss in `loss`: reading the row scales there is rejected."""
    emu = MeasuredEmu()
    with pytest.raises(AssertionError, match=r"cotangent \(row scales\): row \d+"):
        emu.check_measured(emu.run_measured(), scale="loss")


# (call, layer-direction, defect, the row it is seeded into: None where many rows carry it)
DEFECTS = [("loss_grad", "cotangent", "row_scale", 7), ("loss_grad", "cotangent", "pad_row", N_ROWS + 5),
           ("loss_grad", "measured loss", "drop_tile", None),
           ("momentum", "momentum rows", "wrong_row", None), ("momentum", "momentum rows", "unscaled_row", 11),
           ("momentum", "momentum rows", "drop_part", None)]


@pytest.mark.parametrize("what,name,kind,row", DEFECTS)
def test_checker_rejects_a_seeded_measured_defect(what, name, kind, row):
    emu = MeasuredEmu(defect=(name, kind, row if row is not None else 0))
    with pytest.raises(AssertionError, match=re.escape(name) + r".*row %s\b" % (r"\d+" if row is None else row)):
        _run(emu, what)


@pytest.mark.parametrize("pad_scale", [0.0, float("nan")])
def test_checker_rejects_a_scale_applied_to_the_padding_rows(pad_scale):
    """momentum_rows_kernel divides only the real rows by their scale: mscale's tile-padding rows are never written.
    Dividing a padding row's gradient (0) by a scale of 0 or NaN there would put NaN into v and z: seen, naming the row."""
    emu = MeasuredEmu(defect=("momentum rows", "pad_scale", N_ROWS), pad_scale=pad_scale)
    with pytest.raises(AssertionError, match=r"momentum rows \(v\).*row %d\b" % N_ROWS):
        _run(emu, "momentum")


def test_a_scale_applied_to_the_padding_rows_is_harmless_when_finite():
    """With any finite non-zero value in mscale's padding rows the same defect changes no bit (their gradient is 0), so
    no check on the outputs can see it, and none needs to."""
    ws, _ = MeasuredEmu(pad_scale=3.0).run_momentum_rows(LR)
    bad, _ = MeasuredEmu(defect=("momentum rows", "pad_scale", N_ROWS), pad_scale=3.0).run_momentum_rows(LR)
    for k in ("v", "z", "z_h"):
        assert torch.equal(ws[k], bad[k]), k
