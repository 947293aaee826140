"""GPU tests (H100, -m gpu) of the sparse deviations (dgan_reconstruct[_measured[_csr / _conv]]_sparse_dev),
J = D(G(z) + nu) [+ lambda ||z||^2] + l1 ||nu||_1, on MNIST and CelebA, fp32 and fp16 unless noted:
  - step = 0 gives the counterparts' rec, loss and idx bits on the dense, CSR and convolution entries, across
    momentum / Adam, squared error / Huber, prior or not, pruned or not, with dev_out all +0;
  - the unweighted image entry equals the CSR entry on the identity bit for bit at step 0 and 1; w = 1 equals unweighted;
  - the nu update and u against fp32 emulated in numpy on the operands read back from the workspace (0 ulp), and J at
    L = 2 against fp64 on the call's own u, nu and z;
  - R = 10, L = 200 against the fp64 oracle (tests/sparse_dev_oracle.py), image loss and block-average measurements;
  - pruning: keep = R gives the unpruned bits, a schedule the result composed from rec_rr = 1 calls (a prune point
    ranks by J of iteration iter_k - 1, before its update);
  - the header's launch and enqueue counts, and the graph replay of a second call;
  - bad l1, step and dev_out are refused with nothing enqueued;
  - the effect on impulse-noised images of an untrained generator, and DefenseGANBase.rec_sparse_dev."""
import ctypes

import numpy as np
import pytest
import torch

import measured_oracle as MO
import sparse_dev_oracle as S
from gpu_support import gen as _gen, images as _images, option_lr as _lr, read as _read, same as _same, z0 as _z0
from gpu_support import layout, rec as _rec, rec_m as _rec_m, release_cached_memory  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
ADAM = (0.9, 0.999, 1e-8)
CASES = [(p, a) for p in ("fp32", "fp16") for a in ("mnist", "celeba")]


def _identity_csr(n):
    r = torch.arange(n + 1, dtype=torch.int64)
    return torch.sparse_csr_tensor(r, r[:-1], torch.ones(n), (n, n)).cuda()


def _dev(B, arch):
    return torch.full((B,) + SHAPE[arch], float("nan"), device="cuda")


def _zero_bits(t):
    return bool((t.view(torch.int32) == 0).all())


def _sdev_layout(gen, B, R, weighted=0, m=0, nnz=-1, adam=0):
    """Region 0 of an unpruned sparse-deviation workspace (dgan_debug_workspace_layout_sparse_dev)."""
    return layout(gen, "_sparse_dev", B, R, weighted, m, nnz, None, adam, [], 0)[0][0]


# ---- 1. step = 0: the counterparts' bits ----

@pytest.mark.parametrize("precision,arch", CASES)
def test_step_zero_gives_the_counterparts_bits(precision, arch):
    from defensegan_b200.operators import ConvOperator
    B, R, L = 3, 4, 10
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        conv = ConvOperator.box(2)
        yc = conv(x.double()).float()
        kws = (dict(), dict(adam=ADAM), dict(huber_delta=0.05), dict(z_prior=0.1), dict(prune=[(5, 2)]),
               dict(adam=ADAM, huber_delta=0.05, z_prior=0.1, prune=[(2, 3), (6, 1)]))
        for op, ym in ((a, y), (a.to_sparse_csr(), y), (conv, yc)):
            for kw in kws:
                want = _rec_m(gen, ym, op, R, L, _lr(kw), z0, **kw)
                assert bool(torch.isfinite(want[1]).all())
                dev = _dev(B, arch)
                got = _rec_m(gen, ym, op, R, L, _lr(kw), z0, sparse_dev=(0.3, 0.0), deviation_out=dev, **kw)
                assert _same(got, want), (type(op), kw)
                assert _zero_bits(dev), (type(op), kw)
    finally:
        gen.close()


# ---- 2. the image entry is the identity operator ----

@pytest.mark.parametrize("precision,arch", CASES)
def test_image_entry_equals_the_identity_csr_entry(precision, arch):
    B, R, L = 3, 3, 8
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        eye = _identity_csr(n)
        l1 = 0.1 / n
        for kw in (dict(), dict(huber_delta=0.1), dict(adam=ADAM, z_prior=0.05), dict(prune=[(3, 2)])):
            for step in (0.0, 1.0):
                d1, d2, d3 = _dev(B, arch), _dev(B, arch), _dev(B, arch)
                img = _rec(gen, x, R, L, _lr(kw), z0, sparse_dev=(l1, step), deviation_out=d1, **kw)
                csr = _rec_m(gen, x.reshape(B, -1), eye, R, L, _lr(kw), z0, sparse_dev=(l1, step), deviation_out=d2,
                             **kw)
                ones = _rec(gen, x, R, L, _lr(kw), z0, sparse_dev=(l1, step), deviation_out=d3,
                            pixel_weights=torch.ones_like(x), **kw)
                assert bool(torch.isfinite(img[1]).all())
                assert _same(img + [d1], csr + [d2]), (kw, step)
                assert _same(img + [d1], ones + [d3]), (kw, step)
                if step == 1.0:
                    assert float(d1.abs().sum()) > 0, kw
    finally:
        gen.close()


# ---- 3. the update and J on their stored operands ----

def _emulate_update(nu, g, y, eta, tau):
    """fp32 in numpy: a = fmaf(-eta, g, nu) (the fp64 product of two fp32 values is exact, so one rounding is fmaf's),
    nu' = |a| > tau ? a - copysign(tau, a) : +0, u = y + nu'."""
    a = (np.float64(-eta) * g.astype(np.float64) + nu.astype(np.float64)).astype(np.float32)
    t = np.float32(tau)
    nn = np.where(np.abs(a) > t, a - np.copysign(t, a), np.float32(0)).astype(np.float32)
    return nn, (y + nn).astype(np.float32)


@pytest.mark.parametrize("precision,arch", CASES)
def test_update_and_objective_on_stored_operands(precision, arch):
    B, R = 2, 2
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        m = a.shape[0]
        l1, step = 0.05 / n, 1.0
        for measured in (False, True):
            cnt = m if measured else n
            eta = np.float32(step * cnt / 2.0)
            tau = np.float32(np.float64(step) * cnt / 2.0 * np.float64(np.float32(l1)))
            bufs = _sdev_layout(gen, B, R, m=m if measured else 0)
            ws = {}
            for L in (1, 2, 3):
                if measured:
                    _rec_m(gen, y, a, R, L, 0.5, z0, sparse_dev=(l1, step))
                else:
                    _rec(gen, x, R, L, 0.5, z0, sparse_dev=(l1, step))
                ws[L] = {k: _read(gen, bufs, k)[:B * R].cpu().numpy() for k in ("nu", "u", "y", "dym")}
            assert not ws[1]["nu"].view(np.int32).any()
            assert np.array_equal(ws[1]["u"].view(np.int32), ws[1]["y"].view(np.int32))
            # the gradient of iteration t: the image loss writes it every iteration, the measured loop's adjoint
            # product only before an update (so a call of L iterations leaves g_{L-1}, or g_{L-2} measured)
            g = {t: ws[t + (2 if measured else 1)]["dym"] for t in (0, 1)}
            for k in (1, 2):
                nn, uu = _emulate_update(ws[k]["nu"], g[k - 1], ws[k + 1]["y"], eta, tau)
                assert np.array_equal(ws[k + 1]["nu"].view(np.int32), nn.view(np.int32)), (measured, k)
                assert np.array_equal(ws[k + 1]["u"].view(np.int32), uu.view(np.int32)), (measured, k)
            assert (ws[3]["nu"] != 0).any() and (ws[3]["nu"] == 0).any(), measured
        # J at L = 2 against fp64 on the call's own u, nu and z (R = 1: the only restart is returned); the CSR operator
        # (fp32 on both precisions) for the measured loss
        acsr = a.to_sparse_csr()
        for measured in (False, True):
            bufs = _sdev_layout(gen, B, 1, m=m if measured else 0, nnz=acsr.values().numel() if measured else -1)
            if measured:
                _, loss, _ = _rec_m(gen, y, acsr, 1, 2, 0.5, z0[:B], sparse_dev=(l1, step), z_prior=0.1)
            else:
                _, loss, _ = _rec(gen, x, 1, 2, 0.5, z0[:B], sparse_dev=(l1, step), z_prior=0.1)
            u = _read(gen, bufs, "u")[:B].double()
            nu = _read(gen, bufs, "nu")[:B].double()
            z = _read(gen, bufs, "z")[:B, :128].double()
            d = ((u @ a.double().t() - y.double()) ** 2).mean(dim=1) if measured else \
                ((u - x.reshape(B, -1).double()) ** 2).mean(dim=1)
            want = d + float(np.float32(0.1)) * (z * z).sum(dim=1) + float(np.float32(l1)) * nu.abs().sum(dim=1)
            assert float(nu.abs().sum()) > 0
            assert float(((loss.double() - want) / want).abs().max()) <= 1e-5, measured
    finally:
        gen.close()


# ---- 4. the long horizon against the fp64 oracle ----

TOL = {"fp32": (1e-4, 2e-3), "fp16": (3e-2, 1.5e-1)}    # (loss rel. to its scale, rec where the restarts agree)


def _compare(precision, tag, rec, loss, idx, dev, ref, R):
    dl = np.abs(loss.cpu().numpy().astype(np.float64) - ref["loss_min"])
    idx_np = idx.cpu().numpy()
    chosen = ref["loss_all"][np.arange(len(idx_np)) * R + idx_np]
    scale = max(float(np.abs(ref["loss_min"]).max()), 1e-3)
    same = idx_np == ref["idx"]
    drec = np.abs(rec.cpu().numpy().reshape(ref["rec"].shape)[same] - ref["rec"][same]).max() if same.any() else 0.0
    ddev = np.abs(dev.cpu().numpy().reshape(ref["dev"].shape)[same] - ref["dev"][same]).max() if same.any() else 0.0
    print("%s %s: max|dJ| = %.3g (max J %.3g), restart agreement %.2f, max oracle J(chosen) - min %.3g, max|drec| %.3g, "
          "max|dnu| %.3g" % (precision, tag, float(dl.max()), scale, float(same.mean()),
                             float((chosen - ref["loss_min"]).max()), drec, ddev))
    tol = TOL[precision][0] * scale
    assert dl.max() <= tol, tag
    assert float((chosen - ref["loss_min"]).max()) <= tol, tag
    assert drec <= TOL[precision][1] and ddev <= TOL[precision][1], tag


@pytest.mark.parametrize("precision,arch", CASES)
def test_long_horizon_parity_with_the_fp64_oracle(precision, arch):
    """R = 10, L = 200, momentum at rec_lr 10 (the reference's) with step = 1 and tau = 0.1: image loss and 2x2
    block-average measurements (dense)."""
    B, R, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R, 128)
        a = MO.block_average_operator(*SHAPE[arch], 2)
        ym = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        at, xt, yt, z0t = torch.tensor(a).cuda(), torch.tensor(imgs).cuda(), torch.tensor(ym).cuda(), torch.tensor(z0).cuda()
        l1 = 0.2 / n
        ref = S.reconstruct(arch, w, R, L, 10.0, l1, 1.0, images=imgs, z_init_val=z0, device="cuda")
        dev = _dev(B, arch)
        rec, loss, idx = _rec(gen, xt, R, L, 10.0, z0t, sparse_dev=(l1, 1.0), deviation_out=dev)
        _compare(precision, "%s image" % arch, rec, loss, idx, dev, ref, R)
        l1m = 0.2 / a.shape[0]
        ref = S.reconstruct(arch, w, R, L, 10.0, l1m, 1.0, operator=a, measurements=ym, z_init_val=z0, device="cuda")
        dev = _dev(B, arch)
        rec, loss, idx = _rec_m(gen, yt, at, R, L, 10.0, z0t, sparse_dev=(l1m, 1.0), deviation_out=dev)
        _compare(precision, "%s measured dense" % arch, rec, loss, idx, dev, ref, R)
    finally:
        gen.close()


# ---- 5. pruning ----

def _composed(gen, x, R, L, lr, z0, prune, image_shape, measured=None, **kw):
    """The pruned call's result (and dev_out, of image_shape per image) from rec_rr = 1 calls on the tiled images (or
    measurements)."""
    B = x.shape[0]
    xt = x.repeat_interleave(R, dim=0)

    def call(n_it, dev=None):
        if measured is not None:
            return _rec_m(gen, xt, measured, 1, n_it, lr, z0, deviation_out=dev, **kw)
        return _rec(gen, xt, 1, n_it, lr, z0, deviation_out=dev, **kw)
    loss_at = {it: call(it)[1].cpu().numpy() for it, _ in prune}
    dev_all = torch.empty((B * R,) + tuple(image_shape), device="cuda")
    rec_all, loss_all, _ = call(L, dev_all)
    loss_all = loss_all.cpu().numpy()
    rec = torch.empty((B,) + tuple(rec_all.shape[1:]), device="cuda")
    dev = torch.empty((B,) + tuple(image_shape), device="cuda")
    loss, idx = torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
    for i in range(B):
        alive = list(range(R))
        for it, keep in prune:
            ranked = sorted(alive, key=lambda r: (np.isnan(loss_at[it][i * R + r]), loss_at[it][i * R + r], r))
            alive = sorted(ranked[:keep])
        best = alive[0]
        for r in alive[1:]:
            if loss_all[i * R + r] < loss_all[i * R + best]:
                best = r
        rec[i], loss[i], idx[i], dev[i] = rec_all[i * R + best], float(loss_all[i * R + best]), best, dev_all[i * R + best]
    return [rec, loss, idx, dev]


@pytest.mark.parametrize("precision,arch", CASES)
def test_pruning_bit_identities(precision, arch):
    B, R, L = 3, 4, 12
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        for kw in (dict(sparse_dev=(0.1 / n, 1.0)), dict(sparse_dev=(0.1 / n, 0.5), adam=ADAM, huber_delta=0.1)):
            dev = _dev(B, arch)
            plain = _rec(gen, x, R, L, _lr(kw), z0, deviation_out=dev, **kw) + [dev]
            assert bool(torch.isfinite(plain[1]).all())
            for sched in ([(5, R)], [(1, R), (6, R), (11, R)]):
                dev = _dev(B, arch)
                assert _same(_rec(gen, x, R, L, _lr(kw), z0, prune=sched, deviation_out=dev, **kw) + [dev], plain), sched
            for sched in ([(5, 2)], [(3, 3), (6, 2), (9, 1)]):
                dev = _dev(B, arch)
                got = _rec(gen, x, R, L, _lr(kw), z0, prune=sched, deviation_out=dev, **kw) + [dev]
                assert _same(got, _composed(gen, x, R, L, _lr(kw), z0, sched, SHAPE[arch], **kw)), (sched, kw)
            mkw = dict(kw, sparse_dev=(0.1 / a.shape[0], kw["sparse_dev"][1]))
            dev = _dev(B, arch)
            got = _rec_m(gen, y, a, R, L, _lr(kw), z0, prune=[(5, 2)], deviation_out=dev, **mkw) + [dev]
            assert _same(got, _composed(gen, y, R, L, _lr(kw), z0, [(5, 2)], SHAPE[arch], measured=a, **mkw)), kw
    finally:
        gen.close()


# ---- 6. counts ----

@pytest.mark.parametrize("precision,arch", CASES)
def test_launch_and_enqueue_counts(precision, arch):
    from defensegan_b200.operators import ConvOperator
    B, R, L = 2, 3, 9
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        conv = ConvOperator.box(2)
        yc = conv(x.double()).float()
        sd = (0.1 / n, 1.0)
        for kw in (dict(), dict(adam=ADAM, z_prior=0.1), dict(prune=[(3, 2), (6, 1)])):
            P = len(kw.get("prune", []))
            for op, ym in ((a, y), (a.to_sparse_csr(), y), (conv, yc)):
                _rec_m(gen, ym, op, R, L, _lr(kw), z0, **kw)
                base = (gen.last_enqueue_count, gen.last_launch_count)
                for with_dev in (False, True):
                    dev = _dev(B, arch) if with_dev else None
                    for _ in range(2):                      # the second call replays the captured graph
                        _rec_m(gen, ym, op, R, L, _lr(kw), z0, sparse_dev=sd, deviation_out=dev, **kw)
                        assert gen.last_enqueue_count == base[0] + 1 + with_dev, (type(op), kw)
                        assert gen.last_launch_count == base[1] + L + 1 + 2 * P + with_dev, (type(op), kw)
                        assert gen.last_enqueue_count < gen.last_launch_count
            # the image entry: the dense measured sparse-deviation call on the identity, minus its staging and adjoints
            eye = torch.eye(n, device="cuda")
            _rec_m(gen, x.reshape(B, -1), eye, R, L, _lr(kw), z0, sparse_dev=sd, **kw)
            dense = gen.last_launch_count
            del eye
            _rec(gen, x, R, L, _lr(kw), z0, **kw)
            image_enq = gen.last_enqueue_count
            for _ in range(2):
                _rec(gen, x, R, L, _lr(kw), z0, sparse_dev=sd, **kw)
                assert gen.last_launch_count == dense - 3 - (L - 1), kw
                assert gen.last_enqueue_count == image_enq + 1, kw
    finally:
        gen.close()


# ---- 7. refusals ----

@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_bad_arguments_are_refused_with_nothing_enqueued(precision):
    from defensegan_b200 import _native
    B, R, L = 2, 2, 4
    w, gen = _gen("mnist", precision)
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        _rec(gen, x, R, L, 0.5, z0, sparse_dev=(0.001, 1.0))
        before = (gen.last_enqueue_count, gen.last_launch_count)
        ws, need = gen._workspace(B, R, sdev=True)
        prm = _native.dgan_rec_params(B, R, L, 0.5, 0.7, 0, 0, 0)
        out = torch.empty_like(x)
        dev = torch.empty(B * 784 + 4, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        cases = [((-1.0, 1.0), dev, "l1"), ((0.1, float("nan")), dev, "step"), ((float("inf"), 1.0), dev, "l1"),
                 ((0.0, 1e37), dev, "eta"), ((1e36, 1.0), dev, "tau"), ((0.1, 1.0), dev[1:], "dev_out")]
        for (l1, step), d, word in cases:
            sd = _native.dgan_sparse_dev(l1, step)
            rc = gen.lib.dgan_reconstruct_sparse_dev(gen._handle, ctypes.byref(prm), None, None, None, None, 0,
                                                     ctypes.byref(sd), _native._ptr(d), _native._ptr(x), None,
                                                     _native._ptr(z0), _native._ptr(out), None, None, ws, need, stream)
            assert rc == -1, word
            assert word in gen.lib.dgan_last_error().decode(), word
            assert (gen.last_enqueue_count, gen.last_launch_count) == before, word
        rc = gen.lib.dgan_reconstruct_sparse_dev(gen._handle, ctypes.byref(prm), None, None, None, None, 0, None, None,
                                                 _native._ptr(x), None, _native._ptr(z0), _native._ptr(out), None, None,
                                                 ws, need, stream)
        assert rc == -1 and "NULL sparse_dev" in gen.lib.dgan_last_error().decode()
        # the counterpart's checks come first: a misaligned rec_dev is named before a bad l1
        sd = _native.dgan_sparse_dev(-1.0, 1.0)
        rc = gen.lib.dgan_reconstruct_sparse_dev(gen._handle, ctypes.byref(prm), None, None, None, None, 0,
                                                 ctypes.byref(sd), None, _native._ptr(x), None, _native._ptr(z0),
                                                 _native._ptr(dev[1:]), None, None, ws, need, stream)
        assert rc == -1 and "rec_dev" in gen.lib.dgan_last_error().decode()
        torch.cuda.synchronize()
    finally:
        gen.close()


# ---- 8. the effect on impulse noise ----

# Margins set from the first run, on one H100 80GB HBM3 at its 700 W power limit, fp32 and fp16 alike: median error
# 0.2853 without and 0.2805 with deviations on MNIST (ratio 0.983), 2.252 and 2.008 on CelebA (ratio 0.892); the support
# of nu* had precision 1.000 and recall 1.000 on both.  The untrained generator barely depends on z, so the gain is small
# and depends on the draw (tools/sparse_dev_bench.py's 32-image CelebA draw came out worse with deviations).
EFFECT = {"mnist": dict(ratio=0.995, support=0.95), "celeba": dict(ratio=0.95, support=0.95)}


@pytest.mark.parametrize("precision,arch", CASES)
def test_deviations_absorb_impulse_noise(precision, arch):
    """x = G(z_t) with 2 % of its pixels replaced by impulses (the far end of the output range), z0 = z_t + noise, an
    untrained generator: with deviations the median ||G(z*) - G(z_t)|| is lower than without, and nu* covers the spiked
    pixels.  These figures say nothing about a trained generator on real data."""
    B, R, L = 8, 2, 100
    n = HWC[arch]
    w, gen = _gen(arch, precision)
    try:
        g = torch.Generator().manual_seed(21)
        zt = _z0(B, seed=31)
        clean = gen.forward(zt).reshape((B,) + SHAPE[arch]).contiguous()
        lo, hi = (0.0, 1.0) if arch == "mnist" else (-1.0, 1.0)
        spiked = torch.rand(clean.shape, generator=g).cuda() < 0.02
        far = torch.where(clean > (lo + hi) / 2, torch.full_like(clean, lo), torch.full_like(clean, hi))
        x = torch.where(spiked, far, clean)
        z0 = (zt.repeat_interleave(R, dim=0) + 0.3 * torch.randn(B * R, 128, generator=g).cuda()).contiguous()
        tau = 0.25 * (hi - lo)
        sd = (2 * tau / n, 1.0)
        plain, _, _ = _rec(gen, x, R, L, 10.0, z0)
        dev = _dev(B, arch)
        robust, _, _ = _rec(gen, x, R, L, 10.0, z0, sparse_dev=sd, deviation_out=dev)
        e0 = (plain - clean).reshape(B, -1).norm(dim=1).median().item()
        e1 = (robust - clean).reshape(B, -1).norm(dim=1).median().item()
        on = dev != 0
        tp = float((on & spiked).sum())
        precision_ = tp / max(float(on.sum()), 1.0)
        recall = tp / float(spiked.sum())
        print("%s %s: median ||G(z*) - G(z_t)|| %.4g without, %.4g with deviations; nu* support precision %.3f, "
              "recall %.3f" % (precision, arch, e0, e1, precision_, recall))
        assert e1 <= EFFECT[arch]["ratio"] * e0
        assert recall >= EFFECT[arch]["support"] and precision_ >= EFFECT[arch]["support"]
    finally:
        gen.close()


# ---- 9. DefenseGANBase ----

def test_defensegan_rec_sparse_dev_is_the_native_call():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    try:
        gan.rec_rr, gan.rec_iters, gan.rec_lr = 3, 8, 0.5
        gan.rec_sparse_dev = (0.1 / 784, 1.0)
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, 2)).cuda()
        z0 = _z0(6)
        d1, d2 = _dev(2, "mnist"), _dev(2, "mnist")
        got = gan.reconstruct(x, z_init_val=z0, return_aux=True, deviation_out=d1)
        want = gan._native.reconstruct(x, 3, 8, 0.5, z_init_val=z0, sparse_dev=(0.1 / 784, 1.0), deviation_out=d2,
                                       return_aux=True)
        assert _same([t.clone() for t in got] + [d1], [t.clone() for t in want] + [d2])
        assert not _same([t.clone() for t in got], _rec(gan._native, x, 3, 8, 0.5, z0))
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        y = (x.reshape(2, -1).double() @ a.double().t()).float()
        got = gan.reconstruct_measured(y, a, z_init_val=z0, return_aux=True, deviation_out=d1)
        want = gan._native.reconstruct_measured(y, a, 3, 8, 0.5, z_init_val=z0, sparse_dev=(0.1 / 784, 1.0),
                                                deviation_out=d2, return_aux=True)
        assert _same([t.clone() for t in got] + [d1], [t.clone() for t in want] + [d2])
    finally:
        gan.close()
