"""GPU tests (H100, -m gpu) of the projection from convolution measurements (dgan_reconstruct_measured_conv,
dgan_loss_grad_measured_conv) on MNIST and CelebA, both precisions:
  - a shared kernel gives the bits of the CSR call on ConvOperator.to_sparse_csr's matrix: one loop body over a grid of
    geometries, and R = 10, L = 200 projections with and without BatchNorm;
  - per-image kernels give, bit for bit, the single-image CSR calls (momentum, Adam, Huber, a prune schedule);
  - each product against fp64 on the operands it read, read back from the workspace, at 1, 300 and 2560 rows;
  - steady state: no allocation, the documented counts, new kernel values replaying the graph, and conv calls of two
    geometries, CSR, dense and plain calls alternating on one workspace giving fresh handles' bits;
  - bad arguments refused with nothing enqueued."""
import ctypes

import numpy as np
import pytest
import torch

from gpu_support import gen as _gen, layout, release_cached_memory, views  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}


def _taps(kh, kw, seed, zeros=False):
    k = np.random.RandomState(seed).standard_normal((kh, kw)).astype(np.float32) / (kh * kw) ** 0.5
    if zeros and kh * kw > 2:
        k.reshape(-1)[::3] = 0.0
    return k


def _ops():
    """name -> ConvOperator: the host test's geometry grid plus the 5x5 Gaussian and the 2x2 and 4x4 boxes."""
    from defensegan_b200.operators import ConvOperator
    return {
        "even4": ConvOperator(_taps(4, 4, 1), stride=1, padding=1),
        "asym3x5": ConvOperator(_taps(3, 5, 2), stride=2, padding=(0, 2)),
        "stride3": ConvOperator(_taps(5, 3, 3), stride=3, padding=(2, 1)),
        "one": ConvOperator(_taps(1, 1, 4), stride=1, padding=0),
        "zeroneg": ConvOperator(_taps(3, 3, 5, zeros=True), stride=1, padding=1),
        "gauss5": ConvOperator.gaussian(5, 1.0),
        "box2": ConvOperator.box(2),
        "box4": ConvOperator.box(4),
    }


def _measure(op, arch, w, B, seed=2):
    imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=seed)).cuda()
    return op(imgs.double()).float()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_loss_grad_bits_equal_the_csr_call(arch, precision):
    w, gen = _gen(arch, precision)
    try:
        B, R_ = 3, 4
        z = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        for name, op in _ops().items():
            y = _measure(op, arch, w, B)
            csr = op.to_sparse_csr(SHAPE[arch]).cuda()
            want = [t.clone() for t in gen.loss_grad_measured(y, csr, z, R_)]
            got = gen.loss_grad_measured(y, op, z, R_)
            assert bool(torch.isfinite(want[1]).all())
            for what, p, q in zip(("G", "loss", "grad"), want, got):
                assert torch.equal(p, q), (name, what)
            wh = [t.clone() for t in gen.loss_grad_measured(y, csr, z, R_, huber_delta=0.05)]
            gh = gen.loss_grad_measured(y, op, z, R_, huber_delta=0.05)
            for what, p, q in zip(("G", "loss", "grad"), wh, gh):
                assert torch.equal(p, q), (name, "huber", what)
    finally:
        gen.close()


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_reconstruct_bits_equal_the_csr_call(arch, precision, use_bn):
    w, gen = _gen(arch, precision, use_bn)
    try:
        B, R_, L = 2, 10, 200
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        ops = _ops()
        for name in ("gauss5", "box2", "asym3x5"):
            op = ops[name]
            y = _measure(op, arch, w, B)
            lr = 2.0 * (0.05 if use_bn else 1.0)
            csr = op.to_sparse_csr(SHAPE[arch]).cuda()
            want = [t.clone() for t in gen.reconstruct_measured(y, csr, R_, L, lr, z_init_val=z0, return_aux=True)]
            got = gen.reconstruct_measured(y, op, R_, L, lr, z_init_val=z0, return_aux=True)
            assert bool(torch.isfinite(want[1]).all())
            for what, p, q in zip(("rec", "loss", "idx"), want, got):
                assert torch.equal(p, q), (name, what)
    finally:
        gen.close()


@pytest.mark.parametrize("variant", ["momentum", "adam", "huber", "prune"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_per_image_kernels_equal_single_image_csr_calls(arch, precision, variant):
    from defensegan_b200.operators import ConvOperator
    w, gen = _gen(arch, precision)
    try:
        B, R_, L = 3, 4, 60
        ks = np.stack([_taps(5, 5, 10 + i) for i in range(B)])
        op = ConvOperator(ks, stride=2, padding=2)
        y = _measure(op, arch, w, B)
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=5)).cuda()
        kw = {"adam": {"adam": (0.9, 0.999, 1e-8)}, "huber": {"huber_delta": 0.02}, "prune": {"prune": [(40, 2)]},
              "momentum": {}}[variant]
        lr = 0.05 if variant == "adam" else 2.0
        got = [t.clone() for t in gen.reconstruct_measured(y, op, R_, L, lr, z_init_val=z0, return_aux=True, **kw)]
        for i in range(B):
            one = ConvOperator(ks[i], stride=2, padding=2).to_sparse_csr(SHAPE[arch]).cuda()
            want = gen.reconstruct_measured(y[i:i + 1], one, R_, L, lr, z_init_val=z0[i * R_:(i + 1) * R_],
                                            return_aux=True, **kw)
            for what, p, q in zip(("rec", "loss", "idx"), want, got):
                assert torch.equal(p[0], q[i]), (i, what)
    finally:
        gen.close()


def _buffers(gen, n_rows, op):
    """The buffers of the conv-measured workspace of the last call, by name, as views of the workspace."""
    from defensegan_b200 import _native
    kh, kw = op.kernel_size
    cop = _native.dgan_conv_op(kh, kw, op.padding[0], op.padding[1], op.stride)
    return views(gen, layout(gen, "_measured_conv", n_rows, ctypes.byref(cop))[0][0])


@pytest.mark.parametrize("n_rows", [1, 300, 2560])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,name", [("mnist", "stride3"), ("mnist", "gauss5"), ("celeba", "asym3x5")])
def test_each_product_on_its_stored_operands(arch, name, precision, n_rows):
    """r and dy against a float64 conv2d and its autograd adjoint on the operands the kernels read: within 1/2 ulp plus
    (taps + 1) 2^-24 sum |k||operand|; the padded measurements of r and the rows past n_rows exact zeros."""
    from defensegan_b200.operators import ConvOperator
    w, gen = _gen(arch, precision)
    try:
        u = 2.0 ** -24
        base = _ops()[name]
        B = max(1, n_rows // 10)
        R_ = n_rows // B
        kh, kw = base.kernel_size
        ks = base.kernel.unsqueeze(0) * torch.linspace(0.5, 1.5, B).view(B, 1, 1)
        op = ConvOperator(ks, stride=base.stride, padding=base.padding)
        m = op.num_measurements(SHAPE[arch])
        y = _measure(op, arch, w, B) + 0.01 * torch.randn(B, m, generator=torch.Generator().manual_seed(1)).cuda()
        z = torch.tensor(O.sample_z0(n_rows, 128, seed=4)).cuda()
        gen.loss_grad_measured(y, op, z, R_)
        gen._ws.zero_()
        gen.loss_grad_measured(y, op, z, R_)
        torch.cuda.synchronize()
        ws = _buffers(gen, n_rows, op)
        n = n_rows
        assert torch.equal(ws["ck"][:B], ks.reshape(B, -1).cuda())
        k64 = ws["ck"][:B].double().reshape(B, kh, kw).repeat_interleave(R_, dim=0)
        a64 = ConvOperator(k64, stride=op.stride, padding=op.padding)
        absop = ConvOperator(k64.abs(), stride=op.stride, padding=op.padding)
        g = ws["y"][:n].double().reshape((n,) + SHAPE[arch]).requires_grad_(True)
        y_rows = ws["ym"][:B, :m].double().repeat_interleave(R_, dim=0)
        r64 = a64(g) - y_rows
        r = ws["r"][:n].double()
        lim = 0.5 * u * r64.abs() + (kh * kw + 1) * u * (absop(g.detach().abs()) + y_rows.abs()) + 1e-30
        err = (r[:, :m] - r64.detach()).abs()
        assert bool((err <= lim).all()), "r: max err / bound %.3g" % float((err / lim).max())
        assert not ws["r"][:n, m:].any() and not ws["r"][n:].any()
        s32 = float(np.float32(2.0) / np.float32(m))
        (dy64,) = torch.autograd.grad(a64(g), g, grad_outputs=s32 * r[:, :m])
        ga = g.detach().abs().requires_grad_(True)
        (bound,) = torch.autograd.grad(absop(ga), ga, grad_outputs=s32 * r[:, :m].abs())
        dy = ws["dym"][:n].double().reshape(dy64.shape)
        lim_dy = 0.5 * u * dy64.abs() + (kh * kw + 1) * u * bound + 1e-30
        err = (dy - dy64).abs()
        assert bool((err <= lim_dy).all()), "dy: max err / bound %.3g" % float((err / lim_dy).max())
        assert not ws["dym"][n:].any()
        m_ld = ws["r"].shape[1]
        lp = ws["mloss_part"][:, :n].double()
        sq = (r * r).reshape(n, m_ld // 64, 64).sum(dim=2).t()
        assert bool(((lp - sq).abs() <= 8 * u * sq + 1e-30).all())
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_steady_state_replay_and_alternating_calls(precision):
    from defensegan_b200.operators import ConvOperator
    arch, B, R_, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    fresh = []
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        ops = _ops()
        op_a, op_b = ops["gauss5"], ops["stride3"]
        csr = op_a.to_sparse_csr(SHAPE[arch]).cuda()
        dense = csr.to_dense()
        ya, yb = _measure(op_a, arch, w, B), _measure(op_b, arch, w, B)

        def call(g, kind):
            if kind == "conv_a":
                out = g.reconstruct_measured(ya, op_a, R_, L, 1.0, z_init_val=z0, return_aux=True)
            elif kind == "conv_b":
                out = g.reconstruct_measured(yb, op_b, R_, L, 1.0, z_init_val=z0, return_aux=True)
            elif kind in ("csr", "dense"):
                out = g.reconstruct_measured(ya, csr if kind == "csr" else dense, R_, L, 1.0, z_init_val=z0,
                                             return_aux=True)
            else:
                out = g.reconstruct(x, R_, L, 1.0, z_init_val=z0, return_aux=True)
            return [t.clone() for t in out]

        kinds = ("conv_a", "conv_b", "csr", "dense", "plain")
        want = {}
        for kind in kinds:
            _, g = _gen(arch, precision)
            fresh.append(g)
            want[kind] = call(g, kind)
        for kind in kinds + kinds[::-1]:
            for p, q in zip(call(gen, kind), want[kind]):
                assert torch.equal(p, q), kind
        # the documented counts, and a second call at a planned size allocates nothing
        _, plain = _gen(arch, precision)
        fresh.append(plain)
        call(plain, "plain")
        n_plain, e_plain = plain.last_launch_count, plain.last_enqueue_count
        call(gen, "conv_a")
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        call(gen, "conv_a")
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
        per_step = 6 if precision == "fp16" else 3
        assert gen.last_launch_count == n_plain + 1 + per_step * (L - 1) + 1
        assert gen.last_enqueue_count == e_plain
        call(gen, "csr")
        n_csr = gen.last_launch_count
        call(gen, "conv_a")
        assert gen.last_launch_count == n_csr - 4
        # new kernel values and measurements with the same geometry replay the graph and give a fresh handle's bits
        op_c = ConvOperator(_taps(5, 5, 9), stride=1, padding=2)
        yc = _measure(op_c, arch, w, B, seed=7)
        got = [t.clone() for t in gen.reconstruct_measured(yc, op_c, R_, L, 1.0, z_init_val=z0, return_aux=True)]
        assert gen.last_enqueue_count == e_plain
        _, g = _gen(arch, precision)
        fresh.append(g)
        for p, q in zip(got, g.reconstruct_measured(yc, op_c, R_, L, 1.0, z_init_val=z0, return_aux=True)):
            assert torch.equal(p, q)
    finally:
        for g in fresh:
            g.close()
        gen.close()


def test_bad_arguments_are_refused_with_nothing_enqueued():
    from defensegan_b200 import _native
    from defensegan_b200.operators import ConvOperator
    w, gen = _gen("mnist", "fp32")
    try:
        B, R_, L = 2, 3, 5
        op = ConvOperator.gaussian(5, 1.0)
        y = _measure(op, "mnist", w, B)
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        gen.reconstruct_measured(y, op, R_, L, 1.0, z_init_val=z0)
        torch.cuda.synchronize()
        e0 = gen.last_enqueue_count
        k = op.kernels(B, "cuda")
        rec = torch.empty(B * 784 + 4, device="cuda")
        loss = torch.empty(B, device="cuda")
        idx = torch.empty(B, dtype=torch.int32, device="cuda")
        ws, need = gen._workspace(B, R_, conv=_native.dgan_conv_op(5, 5, 2, 2, 1))
        prm = _native.dgan_rec_params(B, R_, L, 1.0, 0.7, 0, 0, 0)
        lib = gen.lib

        def run(cop, kp=k, yp=y, out=rec[:B * 784], sched=None, n_points=0, size=need):
            before = gen.last_enqueue_count
            rc = lib.dgan_reconstruct_measured_conv(gen._handle, ctypes.byref(prm), None, None, sched, n_points,
                                                    ctypes.byref(cop) if cop is not None else None,
                                                    ctypes.c_void_p(kp.data_ptr() if kp is not None else 0),
                                                    ctypes.c_void_p(yp.data_ptr() if yp is not None else 0), None,
                                                    ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(loss.data_ptr()),
                                                    ctypes.c_void_p(idx.data_ptr()), ws, size, None)
            return rc, lib.dgan_last_error().decode(), before

        good = _native.dgan_conv_op(5, 5, 2, 2, 1)
        for cop, word in ((_native.dgan_conv_op(0, 5, 0, 2, 1), "kh"), (_native.dgan_conv_op(5, 33, 2, 2, 1), "kw"),
                          (_native.dgan_conv_op(5, 5, 3, 2, 1), "pad_h"), (_native.dgan_conv_op(5, 5, 2, -1, 1), "pad_w"),
                          (_native.dgan_conv_op(5, 5, 2, 2, 17), "stride")):
            rc, msg, _ = run(cop)
            assert rc == -1 and word in msg, (rc, msg)
        assert run(None)[0] == -1
        assert run(good, kp=None)[0] == -1 and "k_dev" in lib.dgan_last_error().decode()
        assert run(good, yp=None)[0] == -1 and "y_dev" in lib.dgan_last_error().decode()
        assert run(good, out=rec[1:1 + B * 784])[0] == -1
        assert run(good, size=need - 1)[0] == -4
        assert gen.last_enqueue_count == e0          # the count of the last call that ran: the refusals enqueued nothing
        torch.cuda.synchronize()
        assert lib.dgan_conv_op_m(gen._handle, ctypes.byref(good)) == 784
        assert lib.dgan_conv_op_m(gen._handle, ctypes.byref(_native.dgan_conv_op(29, 5, 2, 2, 1))) == 0
    finally:
        gen.close()
    w, gen = _gen("mnist", "fp32", use_bn=True)
    try:
        sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(2, 1))
        cop = _native.dgan_conv_op(5, 5, 2, 2, 1)
        prm = _native.dgan_rec_params(2, 3, 5, 1.0, 0.7, 0, 0, 0)
        k = torch.ones(2, 5, 5, device="cuda")
        y = torch.zeros(2, 784, device="cuda")
        rec = torch.empty(2 * 784, device="cuda")
        rc = gen.lib.dgan_reconstruct_measured_conv(gen._handle, ctypes.byref(prm), None, None, sched, 1,
                                                    ctypes.byref(cop), ctypes.c_void_p(k.data_ptr()),
                                                    ctypes.c_void_p(y.data_ptr()), None, ctypes.c_void_p(rec.data_ptr()),
                                                    None, None, ctypes.c_void_p(rec.data_ptr()), 1 << 30, None)
        assert rc == -3
    finally:
        gen.close()
